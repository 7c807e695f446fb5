"""ctypes binding of libowshen_b200.so and the host-side mirror of the API BASELINE.json's north_star
names: prove() / verify() / MerkleTree.  The reference (OwshenNetwork/owshen @ c7b1f00) has no such
API (SURVEY.md section 0), so names and error behaviour follow its conventions instead: fallible
calls raise (anyhow::Result -> exception), byte blobs are owned `bytes`, field elements are 32-byte
little-endian (/root/reference/src/blockchain/tx/owshen_airdrop/babyjubjub/mod.rs:7-11).

All hashing, witness generation, NTTs and MSMs run in the CUDA library; nothing here computes.
"""
import array
import bisect
import ctypes as C
import os
import secrets as _rand
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
# OWSHEN_B200_LIB: an alternative build of the same library (A/B experiments of compile-time variants)
_LIB_PATH = os.environ.get("OWSHEN_B200_LIB") or os.path.join(_HERE, "libowshen_b200.so")
_lib = None

FR_MODULUS = 21888242871839275222246405745257275088548364400416034343698204186575808495617
PROOF_BYTES = 256

OG_OK, OG_E_INVALID, OG_E_VERIFY = 0, -1, -6

# encrypted notes: l, the prime order of the BabyJubJub BASE (view keys and ephemerals must be nonzero mod l), and the two
# owner sentinels of note_scan
NOTE_SUBGROUP_ORDER = 2736030358979909402780800718157159386076813972158567259200215660948447373041
NOTE_NOT_OWNED, NOTE_MALFORMED = 0xFFFFFFFF, 0xFFFFFFFE
NOTE_RECORD_BYTES, NOTE_PLAINTEXT_BYTES = 160, 128


class OwshenB200Error(RuntimeError):
    def __init__(self, code, detail=""):
        self.code = code
        msg = lib().og_strerror(code).decode() if _lib is not None else str(code)
        super().__init__(f"owshen_b200 error {code}: {msg}" + (f" ({detail})" if detail else ""))


def build_library(jobs=8):
    """Compile every CUDA source for sm_90a into owshen_b200/libowshen_b200.so (in-tree)."""
    subprocess.run(["make", "-C", os.path.join(_HERE, "csrc"), f"-j{jobs}"], check=True, stdout=subprocess.DEVNULL)


_u8p = C.c_char_p
_SIGS = {
    "og_abi_version": (C.c_int32, []),
    "og_strerror": (C.c_char_p, [C.c_int32]),
    "og_last_error": (C.c_char_p, [C.c_void_p]),
    "og_init": (C.c_int32, [C.c_int32, C.POINTER(C.c_void_p)]),
    "og_free": (None, [C.c_void_p]),
    "og_sync": (C.c_int32, [C.c_void_p]),
    "og_stream": (C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "og_timer_start": (C.c_int32, [C.c_void_p]),
    "og_timer_stop": (C.c_int32, [C.c_void_p, C.POINTER(C.c_float)]),
    "og_launch_count": (C.c_uint64, [C.c_void_p]),
    "og_profile": (C.c_int32, [C.c_void_p, C.c_int32]),
    "og_profile_dump": (C.c_int32, [C.c_void_p, C.c_char_p, C.c_uint64]),
    "og_imad_peak": (C.c_int32, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "og_int_pipe_peaks": (C.c_int32, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "og_mul_latency": (C.c_int32, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "og_hybrid_probe": (C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    "og_fp64_peak": (C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    "og_field_op": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_mimc7_constants": (C.c_int32, [C.c_void_p, C.POINTER(C.c_uint32)]),
    "og_mimc7_hash2": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_mimc7_merkle_paths": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "og_mimc7_merkle_paths_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "og_mimc7_merkle_build": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_mimc7_merkle_append": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_bjj_verify_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p]),
    "og_bjj_verify_batch_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p]),
    "og_bjj_sign_batch_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_bjj_sign_batch": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_note_public_keys": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "og_note_encrypt": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 7 + [C.c_uint64] + [C.c_void_p] * 3),
    "og_note_encrypt_dev": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 7 + [C.c_uint64] + [C.c_void_p] * 3),
    "og_note_scan": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "og_note_scan_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "og_owned_note_encrypt": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 7 + [C.c_uint64] + [C.c_void_p] * 3),
    "og_owned_note_encrypt_dev": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 7 + [C.c_uint64] + [C.c_void_p] * 3),
    "og_owned_note_scan": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                       C.c_void_p]),
    "og_owned_note_scan_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                           C.c_void_p]),
    "og_owned_labeled_note_encrypt": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 8 + [C.c_uint64] + [C.c_void_p] * 3),
    "og_owned_labeled_note_encrypt_dev": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 8 + [C.c_uint64] + [C.c_void_p] * 3),
    "og_owned_labeled_note_scan": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64,
                                               C.c_void_p, C.c_void_p]),
    "og_owned_labeled_note_scan_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64,
                                                   C.c_void_p, C.c_void_p]),
    "og_msm_g1": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_msm_g2": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_msm_g1_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_msm_g2_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g1_generator_mul": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g2_generator_mul": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g1_generator_mul_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g2_generator_mul_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g1_sum_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g2_sum_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g1_sum": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_g2_sum": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_ntt": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32]),
    "og_ntt_dev": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32]),
    "og_withdraw_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_withdraw_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_withdraw_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p]),
    "og_deposit_r1cs_info": (C.c_int32, [C.POINTER(C.c_uint32)] * 4),
    "og_deposit_r1cs_export": (C.c_int32, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_deposit_witness": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 3 + [C.c_uint32, C.c_void_p]),
    "og_transfer_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_transfer_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_transfer_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 11 + [C.c_uint32, C.c_void_p]),
    "og_association_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_association_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_association_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 7 + [C.c_uint32, C.c_void_p]),
    "og_exclusion_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_exclusion_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_exclusion_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 9 + [C.c_uint32, C.c_void_p]),
    "og_labeled_precommitments": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_labeled_leaves": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p]),
    "og_labeled_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_labeled_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_labeled_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 15 + [C.c_uint32, C.c_void_p]),
    "og_labeled_association_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_labeled_association_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_labeled_association_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 13 + [C.c_uint32, C.c_void_p]),
    "og_owned_public_keys": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "og_owned_commitments": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p]),
    "og_owned_nullifiers": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 3 + [C.c_uint64, C.c_void_p]),
    "og_owned_transfer_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_owned_transfer_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_owned_transfer_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 11 + [C.c_uint32, C.c_void_p]),
    "og_owned_labeled_precommitments": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 2 + [C.c_uint64, C.c_void_p]),
    "og_owned_labeled_leaves": (C.c_int32, [C.c_void_p] + [C.c_void_p] * 4 + [C.c_uint64, C.c_void_p]),
    "og_owned_labeled_transfer_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_owned_labeled_transfer_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_owned_labeled_transfer_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 15 + [C.c_uint32, C.c_void_p]),
    "og_ragequit_r1cs_info": (C.c_int32, [C.c_uint32] + [C.POINTER(C.c_uint32)] * 4),
    "og_ragequit_r1cs_export": (C.c_int32, [C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_ragequit_witness": (C.c_int32, [C.c_void_p, C.c_uint32] + [C.c_void_p] * 9 + [C.c_uint32, C.c_void_p]),
    "og_groth16_setup_withdraw": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_groth16_setup": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32] + [C.c_void_p] * 9
                         + [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_load_pk": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]),
    "og_free_pk": (None, [C.c_void_p]),
    "og_pk_info": (C.c_int32, [C.c_void_p] + [C.POINTER(C.c_uint32)] * 4),
    "og_pk_window_bits": (C.c_int32, [C.c_void_p, C.POINTER(C.c_uint32)]),
    "og_groth16_prove": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_withdraw": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_withdraw_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_deposit": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 3 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_deposit_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 3 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_transfer": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 11 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_transfer_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 11 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_association": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 7 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_association_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 7 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_exclusion": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 9 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_exclusion_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 9 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_labeled": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 15 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_labeled_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 15 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_labeled_association": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 13 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_labeled_association_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 13
                                                 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_owned_transfer": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 11 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_owned_transfer_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 11
                                            + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_owned_labeled_transfer": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 15
                                                + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_owned_labeled_transfer_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 15
                                                    + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_ragequit": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 9 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_prove_ragequit_dev": (C.c_int32, [C.c_void_p, C.c_void_p] + [C.c_void_p] * 9 + [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_pk_prover_plan": (C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]),
    "og_groth16_h_evals": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "og_groth16_verify": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p]),
    "og_ptau_new": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_ptau_contribute": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_ptau_verify": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]),
    "og_ptau_prepare": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32] + [C.c_void_p] * 9
                        + [C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_ptau_prepare_withdraw": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                             C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_phase2_contribute": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.POINTER(C.c_uint64), C.c_void_p, C.POINTER(C.c_uint64),
                                         C.c_void_p, C.POINTER(C.c_uint64)]),
    "og_phase2_verify": (C.c_int32, [C.c_void_p] + [C.c_void_p, C.c_uint64] * 5),
    "og_scale_points": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p]),
    "og_intt_points": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint32]),
    "og_msm_bucket_sums": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                       C.c_uint64, C.c_int32, C.c_void_p, C.c_void_p]),
    "og_field_probe_raw": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
}
ABI_SYMBOLS = tuple(_SIGS)


def lib():
    """Load libowshen_b200.so; raises if the CUDA extension has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise OSError(f"{_LIB_PATH} is missing: build it with owshen_b200.build_library() / "
                          "`make -C owshen_b200/csrc` -- there is no CPU fallback")
        L = C.CDLL(_LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _check(rc, ctx=None):
    if rc != OG_OK:
        detail = ""
        if ctx is not None and ctx._h:
            detail = lib().og_last_error(ctx._h).decode(errors="replace")
        raise OwshenB200Error(rc, detail)


def _ptr(x):
    """bytes / bytearray / int address / object with .ctypes or data_ptr() -> void*"""
    if x is None:
        return None
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, (bytes, bytearray)):
        return C.cast(C.c_char_p(bytes(x)) if isinstance(x, bytearray) else C.c_char_p(x), C.c_void_p)
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    if hasattr(x, "ctypes"):
        return C.c_void_p(x.ctypes.data)
    return C.cast(x, C.c_void_p)


def _need(cond, what):
    """Argument validation at the Python boundary: the C side takes plain pointers and trusts the sizes it is given,
    so every wrapper checks lengths first and raises ValueError (never `assert`, which python -O strips)."""
    if not cond:
        raise ValueError(what)


def _blen(x):
    """Byte length of a bytes-like / array / tensor argument, or None when only an address was passed."""
    if isinstance(x, (bytes, bytearray, memoryview)):
        return len(x)
    if hasattr(x, "nbytes"):
        return int(x.nbytes)
    if hasattr(x, "numel") and hasattr(x, "element_size"):
        return int(x.numel() * x.element_size())
    return None


def _need_len(x, n, name):
    got = _blen(x)
    _need(got is None or got == n, f"{name}: expected {n} bytes, got {got}")


def _bits_array(bits):
    return (C.c_uint32 * len(bits))(*[int(b) & 0xFFFFFFFF for b in bits])


def _u64_array(xs):
    """Amounts as a buffer of little-endian uint64: bytes-like, a uint64 array / tensor, or a sequence of ints < 2^64."""
    if _blen(xs) is not None or isinstance(xs, int):
        return xs
    vals = [int(x) for x in xs]
    _need(all(0 <= x < 1 << 64 for x in vals), "amounts must be integers in [0, 2^64)")
    return (C.c_uint64 * len(vals))(*vals)


def _u32_array(xs):
    return xs if _blen(xs) is not None or isinstance(xs, int) else _bits_array(xs)


def _label_array(xs):
    """Labels as a buffer of little-endian uint32: bytes-like, a uint32 array / tensor, or a sequence of ints < 2^32."""
    if _blen(xs) is not None or isinstance(xs, int):
        return xs
    vals = [int(x) for x in xs]
    _need(all(0 <= x < 1 << 32 for x in vals), "labels must be integers in [0, 2^32)")
    return (C.c_uint32 * len(vals))(*vals)


# The statements' boundary, mirroring the statement table of csrc/mimc.cuh: statement -> (takes a depth, input arrays in C ABI
# order as (name, bytes per proof, bytes per proof and tree level, conversion of a sequence of ints)).  The C entry points are
# og_<statement>_r1cs_info / _r1cs_export / _witness and og_groth16_prove_<statement>(_dev).
_STATEMENTS = {
    "withdraw": (True, (("nullifiers", 32, 0, None), ("secrets", 32, 0, None), ("recipients", 32, 0, None), ("siblings", 0, 32, None),
                        ("path_bits", 4, 0, _u32_array))),
    "deposit": (False, (("nullifiers", 32, 0, None), ("secrets", 32, 0, None), ("depositors", 32, 0, None))),
    "transfer": (True, (("roots", 32, 0, None), ("tokens", 32, 0, None), ("recipients", 32, 0, None), ("in_nullifiers", 64, 0, None),
                        ("in_secrets", 64, 0, None), ("in_amounts", 16, 0, _u64_array), ("in_siblings", 0, 64, None),
                        ("in_path_bits", 8, 0, _u32_array), ("out_nullifiers", 64, 0, None), ("out_secrets", 64, 0, None),
                        ("out_amounts", 16, 0, _u64_array))),
    "association": (True, (("nullifiers", 32, 0, None), ("secrets", 32, 0, None), ("recipients", 32, 0, None), ("siblings", 0, 32, None),
                           ("path_bits", 4, 0, _u32_array), ("assoc_siblings", 0, 32, None), ("assoc_path_bits", 4, 0, _u32_array))),
    "exclusion": (True, (("nullifiers", 32, 0, None), ("secrets", 32, 0, None), ("recipients", 32, 0, None), ("siblings", 0, 32, None),
                         ("path_bits", 4, 0, _u32_array), ("excl_low", 8, 0, _u64_array), ("excl_next", 8, 0, _u64_array),
                         ("excl_siblings", 0, 32, None), ("excl_path_bits", 4, 0, _u32_array))),
    "labeled": (True, (("tokens", 32, 0, None), ("recipients", 32, 0, None), ("withdrawn", 8, 0, _u64_array), ("nullifiers", 32, 0, None),
                       ("secrets", 32, 0, None), ("amounts", 8, 0, _u64_array), ("labels", 4, 0, _label_array), ("siblings", 0, 32, None),
                       ("path_bits", 4, 0, _u32_array), ("change_nullifiers", 32, 0, None), ("change_secrets", 32, 0, None),
                       ("excl_low", 8, 0, _u64_array), ("excl_next", 8, 0, _u64_array), ("excl_siblings", 0, 32, None),
                       ("excl_path_bits", 4, 0, _u32_array))),
    "labeled_association": (True, (("tokens", 32, 0, None), ("recipients", 32, 0, None), ("withdrawn", 8, 0, _u64_array),
                                   ("nullifiers", 32, 0, None), ("secrets", 32, 0, None), ("amounts", 8, 0, _u64_array),
                                   ("labels", 4, 0, _label_array), ("siblings", 0, 32, None), ("path_bits", 4, 0, _u32_array),
                                   ("change_nullifiers", 32, 0, None), ("change_secrets", 32, 0, None), ("assoc_siblings", 0, 32, None),
                                   ("assoc_path_bits", 4, 0, _u32_array))),
    "owned_transfer": (True, (("roots", 32, 0, None), ("tokens", 32, 0, None), ("recipients", 32, 0, None), ("in_spend_keys", 64, 0, None),
                              ("in_blindings", 64, 0, None), ("in_amounts", 16, 0, _u64_array), ("in_siblings", 0, 64, None),
                              ("in_path_bits", 8, 0, _u32_array), ("out_owners", 64, 0, None), ("out_blindings", 64, 0, None),
                              ("out_amounts", 16, 0, _u64_array))),
    "owned_labeled_transfer": (True, (("roots", 32, 0, None), ("tokens", 32, 0, None), ("recipients", 32, 0, None),
                                      ("withdrawn", 8, 0, _u64_array), ("labels", 4, 0, _label_array), ("in_spend_keys", 64, 0, None),
                                      ("in_blindings", 64, 0, None), ("in_amounts", 16, 0, _u64_array), ("in_siblings", 0, 64, None),
                                      ("in_path_bits", 8, 0, _u32_array), ("out_owners", 64, 0, None), ("out_blindings", 64, 0, None),
                                      ("out_amounts", 16, 0, _u64_array), ("assoc_siblings", 0, 32, None),
                                      ("assoc_path_bits", 4, 0, _u32_array))),
    "ragequit": (True, (("roots", 32, 0, None), ("tokens", 32, 0, None), ("recipients", 32, 0, None), ("amounts", 8, 0, _u64_array),
                        ("labels", 4, 0, _label_array), ("spend_keys", 32, 0, None), ("blindings", 32, 0, None), ("siblings", 0, 32, None),
                        ("path_bits", 4, 0, _u32_array))),
}


def _depth_arg(stmt, depth):
    """The depth argument of statement `stmt`'s C entry points: [depth], or [] for a statement of one fixed shape."""
    return [depth] if _STATEMENTS[stmt][0] else []


def _batch_args(fn, columns, sizes, arrays):
    """Length checks of a batch's input arrays (sequences of ints converted first) -> their pointers in C ABI order: array k
    is columns[k] = (name, ..., conversion of a sequence of ints) and must hold sizes[k] bytes."""
    out = []
    for (name, *_, conv), size, buf in zip(columns, sizes, arrays):
        buf = conv(buf) if conv else buf
        if isinstance(buf, C.Array):        # converted from a sequence
            _need(C.sizeof(buf) == size, f"{fn}: {name}: expected {size // C.sizeof(buf._type_)} values, got {len(buf)}")
        else:
            _need_len(buf, size, f"{fn}: {name}")
        out.append(_ptr(buf))
    return out


def _statement_args(stmt, fn, batch, depth, arrays):
    """_batch_args of statement `stmt`'s input arrays for `batch` proofs at `depth`."""
    columns = _STATEMENTS[stmt][1]
    return _batch_args(fn, columns, [(per_proof + per_level * depth) * batch for _, per_proof, per_level, _ in columns], arrays)


# The note hashes' boundary, mirroring the note-hash table of csrc/mimc.cuh: hash -> its columns in C ABI order as (name, bytes
# per item, conversion of a sequence of ints).  The C entry point is og_<hash>, and Context.<hash> wraps it.
_NOTE_HASHES = {
    "labeled_precommitments": (("nullifiers", 32, None), ("secrets", 32, None)),
    "labeled_leaves": (("precommitments", 32, None), ("tokens", 32, None), ("amounts", 8, _u64_array), ("labels", 4, _label_array)),
    "owned_public_keys": (("spend_keys", 32, None),),
    "owned_commitments": (("owners", 32, None), ("blindings", 32, None), ("tokens", 32, None), ("amounts", 8, _u64_array)),
    "owned_nullifiers": (("spend_keys", 32, None), ("commitments", 32, None), ("indices", 4, _label_array)),
    "owned_labeled_precommitments": (("owners", 32, None), ("blindings", 32, None)),
    "owned_labeled_leaves": (("precommitments", 32, None), ("tokens", 32, None), ("amounts", 8, _u64_array), ("labels", 4, _label_array)),
}


# The note kinds' encryption inputs in C ABI order, as (name, bytes per note, conversion of a sequence of ints); the C entry
# points are og_<kind>_encrypt(_dev) and og_<kind>_scan(_dev), the owned kinds' scans taking a spend public key per view key.
_NOTE_KINDS = {
    "note": (("pk_x", 32, None), ("pk_is_odd", 1, None), ("nullifiers", 32, None), ("secrets", 32, None), ("tokens", 32, None),
             ("amounts", 8, _u64_array), ("ephemerals", 32, None)),
    "owned_note": (("pk_x", 32, None), ("pk_is_odd", 1, None), ("owners", 32, None), ("blindings", 32, None), ("tokens", 32, None),
                   ("amounts", 8, _u64_array), ("ephemerals", 32, None)),
    "owned_labeled_note": (("pk_x", 32, None), ("pk_is_odd", 1, None), ("owners", 32, None), ("blindings", 32, None),
                           ("tokens", 32, None), ("amounts", 8, _u64_array), ("labels", 4, _label_array), ("ephemerals", 32, None)),
}


def _note_keys(fn, view_keys, spend_public_keys):
    """The key arguments of a scan: the view keys, the spend public keys unless None (transfer notes), and the key count."""
    if spend_public_keys is None:
        _need(len(view_keys) % 32 == 0, f"{fn}: view keys must be a multiple of 32 bytes")
        return [view_keys, len(view_keys) // 32]
    _need(len(view_keys) % 32 == 0 and len(spend_public_keys) == len(view_keys),
          f"{fn}: view keys and spend public keys must be equally long multiples of 32 bytes")
    return [view_keys, spend_public_keys, len(view_keys) // 32]


def fr_bytes(x: int) -> bytes:
    return (x % FR_MODULUS).to_bytes(32, "little")


class Context:
    """One CUDA device + one stream (og_ctx)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        _check(lib().og_init(device, C.byref(self._h)))
        self.device = device

    def close(self):
        if getattr(self, "_h", None) and _lib is not None:
            _lib.og_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown
            pass

    def sync(self):
        _check(lib().og_sync(self._h), self)

    @property
    def cuda_stream(self) -> int:
        """Address of the cudaStream_t the `_dev` entry points enqueue on (wrap with torch.cuda.ExternalStream)."""
        p = C.c_void_p()
        _check(lib().og_stream(self._h, C.byref(p)), self)
        return p.value or 0

    def timer_start(self):
        _check(lib().og_timer_start(self._h), self)

    def timer_stop(self) -> float:
        ms = C.c_float()
        _check(lib().og_timer_stop(self._h, C.byref(ms)), self)
        return ms.value

    @property
    def launch_count(self) -> int:
        return lib().og_launch_count(self._h)

    def profile(self, enable: bool):
        _check(lib().og_profile(self._h, int(enable)), self)

    def profile_dump(self) -> dict:
        """{kernel: (launches, total_ms)} since the previous dump (synchronises the stream)."""
        buf = C.create_string_buffer(1 << 16)
        _check(lib().og_profile_dump(self._h, buf, len(buf)), self)
        out = {}
        for line in buf.value.decode().splitlines():
            name, n, ms = line.rsplit(",", 2)
            out[name] = (int(n), float(ms))
        return out

    def imad_peak(self):
        a, b = C.c_double(), C.c_double()
        _check(lib().og_imad_peak(self._h, C.byref(a), C.byref(b)), self)
        return a.value, b.value

    def mul_latency(self):
        a, b = C.c_double(), C.c_double()
        _check(lib().og_mul_latency(self._h, C.byref(a), C.byref(b)), self)
        return a.value, b.value

    def hybrid_probe(self) -> dict:
        r = (C.c_double * 4)()
        _check(lib().og_hybrid_probe(self._h, r), self)
        return {"fp64_products_52bit_alone": r[0], "imad_wide_chain_alone": r[1],
                "fp64_products_52bit_mixed": r[2], "imad_wide_chain_mixed": r[3]}

    def fp64_peak(self) -> float:
        v = C.c_double()
        _check(lib().og_fp64_peak(self._h, C.byref(v)), self)
        return v.value

    def int_pipe_peaks(self) -> dict:
        a, b, c = C.c_double(), C.c_double(), C.c_double()
        _check(lib().og_int_pipe_peaks(self._h, C.byref(a), C.byref(b), C.byref(c)), self)
        return {"imad_per_s": a.value, "imad_wide_per_s": b.value, "imad_wide_carry_chain_per_s": c.value}

    # ---- probes / kernels on host buffers -------------------------------------------------------
    def field_op(self, field: str, op: str, a: bytes, b: bytes) -> bytes:
        _need(len(a) % 32 == 0 and len(b) == len(a), "field_op: a and b must be equally long multiples of 32 bytes")
        _need(field in ("fq", "fr") and op in ("mul", "add", "sub"), "field_op: unknown field or op")
        n = len(a) // 32
        out = C.create_string_buffer(32 * n)
        _check(lib().og_field_op(self._h, {"fq": 0, "fr": 1}[field], {"mul": 0, "add": 1, "sub": 2}[op], a, b, n, out), self)
        return out.raw

    # ops of field_probe_raw per unit (include/owshen_b200.h: og_field_probe_raw)
    FIELD_PROBE_OPS = {"g1": ("mul", "sqr", "sub", "dbl", None, None, None, None,
                              "mul_lazy", "sqr_lazy", "add_lazy", "sub_lazy", "canonical", "is_zero_lazy", "mul_sum_lazy"),
                       "g2": ("mul_lazy", "sqr_lazy", "add_lazy", "sub_lazy", "canonical", "mul", "sqr", "is_zero_lazy")}

    def field_probe_raw(self, unit: str, op: str, a: bytes, b: bytes = None) -> bytes:
        """Test/debug probe: element-wise arithmetic of the G1 ("g1": Fq, 32 B per operand) or G2 ("g2": Fq2, 64 B) MSM unit on
        raw Montgomery limbs, through the functions its bucket kernels call (the probe kernel's own compiled copies); raw limbs out."""
        _need(unit in self.FIELD_PROBE_OPS and op is not None and op in self.FIELD_PROBE_OPS[unit], "field_probe_raw: unknown unit or op")
        eb = 32 if unit == "g1" else 64
        b = a if b is None else b
        _need(len(a) % eb == 0 and len(b) == len(a), f"field_probe_raw: a and b must be equally long multiples of {eb} bytes")
        n = len(a) // eb
        out = C.create_string_buffer(eb * n)
        _check(lib().og_field_probe_raw(self._h, unit == "g2", self.FIELD_PROBE_OPS[unit].index(op), a, b, n, out), self)
        return out.raw

    def msm_bucket_sums(self, curve: str, points: bytes, counts, entries, n_groups: int, nb: int, n_entries_max=None,
                        few_groups=False, buckets=False):
        """Test/debug probe (og_msm_bucket_sums): the MSM engine's bucket stage on the given bucket lists.  counts: n_groups * nb
        list lengths (key = g * nb + b); entries: sum(counts) words (point index << 1) | negate in key order; n_entries_max
        (default sum(counts)) sets the heavy-bucket cap as in the MSM.  Returns (n_groups affine totals sum_b (b + 1) B_b, the
        n_groups * nb affine buckets or None)."""
        _need(curve in ("g1", "g2"), "msm_bucket_sums: curve must be 'g1' or 'g2'")
        pb = 64 if curve == "g1" else 128
        _need(len(points) % pb == 0, f"msm_bucket_sums: points must be a multiple of {pb} bytes")
        def u32(xs):                       # a sequence of ints or a numpy array -> a buffer of uint32
            if not hasattr(xs, "astype"):
                return array.array("I", xs)
            a = array.array("I")
            a.frombytes(xs.astype("<u4").tobytes())
            return a
        cnt, ent = u32(counts), u32(entries)
        total = sum(cnt)
        _need(len(cnt) == n_groups * nb and len(ent) == total, "msm_bucket_sums: need n_groups * nb counts and sum(counts) entries")
        out = C.create_string_buffer(pb * n_groups)
        bk = C.create_string_buffer(pb * n_groups * nb) if buckets else None
        _check(lib().og_msm_bucket_sums(self._h, curve == "g2", points, len(points) // pb, C.c_void_p(cnt.buffer_info()[0]),
                                        C.c_void_p(ent.buffer_info()[0]) if total else None, n_groups, nb,
                                        total if n_entries_max is None else n_entries_max, int(few_groups), out, bk), self)
        return out.raw, (bk.raw if buckets else None)

    def mimc7_hash2(self, left: bytes, right: bytes) -> bytes:
        _need(len(left) % 32 == 0 and len(right) == len(left), "mimc7_hash2: left and right must be equally long multiples of 32 bytes")
        n = len(left) // 32
        out = C.create_string_buffer(32 * n)
        _check(lib().og_mimc7_hash2(self._h, left, right, n, out), self)
        return out.raw

    def merkle_paths(self, leaves: bytes, siblings: bytes, path_bits, depth: int) -> bytes:
        _need(0 <= depth <= 32 and len(leaves) % 32 == 0, "merkle_paths: depth must be <= 32 and leaves a multiple of 32 bytes")
        n = len(leaves) // 32
        _need(len(siblings) == 32 * n * depth and len(path_bits) == n, "merkle_paths: siblings must hold n*depth elements and path_bits n words")
        out = C.create_string_buffer(32 * n * (depth + 1))
        _check(lib().og_mimc7_merkle_paths(self._h, leaves, siblings, _bits_array(path_bits), n, depth, out), self)
        return out.raw

    def merkle_build(self, leaves: bytes) -> bytes:
        _need(len(leaves) % 32 == 0 and len(leaves) >= 32, "merkle_build: leaves must be a non-empty multiple of 32 bytes")
        n = len(leaves) // 32
        _need(n & (n - 1) == 0, "merkle_build: the leaf count must be a power of two (pad with empty leaves)")
        out = C.create_string_buffer(32 * (2 * n - 1))
        _check(lib().og_mimc7_merkle_build(self._h, leaves, n, out), self)
        return out.raw

    def merkle_append(self, depth: int, start: int, leaves: bytes, left_boundary: bytes, zeros: bytes) -> bytes:
        """Nodes of levels 1..depth touched by appending len(leaves)/32 leaves at index `start` (og_mimc7_merkle_append)."""
        _need(1 <= depth <= 32 and len(leaves) % 32 == 0 and len(leaves) > 0, "merkle_append: bad depth or leaves")
        n = len(leaves) // 32
        _need(start >= 0 and start + n <= (1 << depth), "merkle_append: the leaves do not fit the tree")
        _need(len(left_boundary) == 32 * depth and len(zeros) == 32 * depth, "merkle_append: boundary and zeros hold one element per level")
        total = sum(((start + n - 1) >> l) - (start >> l) + 1 for l in range(1, depth + 1))
        out = C.create_string_buffer(32 * total)
        _check(lib().og_mimc7_merkle_append(self._h, depth, start, leaves, n, left_boundary, zeros, out), self)
        return out.raw

    def bjj_verify_batch(self, pk_x: bytes, pk_is_odd: bytes, messages: bytes, signatures: bytes, hash_kind: int = 0) -> bytes:
        """BabyJubJub batch verification; one status byte per signature (1 ok, 0 bad, 2 undecompressible pk)."""
        n = len(pk_is_odd)
        _need(len(pk_x) == 32 * n and len(messages) == 32 * n and len(signatures) == 96 * n, "bjj_verify_batch: inconsistent lengths")
        _need(hash_kind in (0, 1), "bjj_verify_batch: hash_kind must be 0 or 1")
        out = C.create_string_buffer(n)
        _check(lib().og_bjj_verify_batch(self._h, pk_x, pk_is_odd, messages, signatures, n, hash_kind, out), self)
        return out.raw

    def bjj_sign_batch(self, secret_keys: bytes, randomness: bytes, messages: bytes, hash_kind: int = 0):
        """BabyJubJub key derivation + signing, one key per 32 bytes: -> (pk_x, pk_is_odd, signatures, status) with
        status 1 = signed, 2 = the reference's sign() would return Err("Invalid repr")."""
        _need(len(secret_keys) % 32 == 0 and len(randomness) == len(secret_keys) and len(messages) == len(secret_keys),
              "bjj_sign_batch: keys, randomness and messages must be equally long multiples of 32 bytes")
        _need(hash_kind in (0, 1), "bjj_sign_batch: hash_kind must be 0 or 1")
        n = len(secret_keys) // 32
        px, odd = C.create_string_buffer(32 * n), C.create_string_buffer(n)
        sg, st = C.create_string_buffer(96 * n), C.create_string_buffer(n)
        _check(lib().og_bjj_sign_batch(self._h, secret_keys, randomness, messages, n, hash_kind, px, odd, sg, st), self)
        return px.raw, odd.raw[:n], sg.raw, st.raw[:n]

    # ---- encrypted notes: one encryption and one scan for every note kind (_NOTE_KINDS) -----------------------------------
    def _note_encrypt(self, kind, arrays):
        """og_<kind>_encrypt of the notes in `arrays` (_NOTE_KINDS[kind] order, one note per pk_is_odd byte), ephemerals drawn
        with the `secrets` module in [1, l) when None -> (records, commitments, status)."""
        n = len(arrays[1])
        if arrays[-1] is None:
            arrays = (*arrays[:-1], b"".join(fr_bytes(_rand.randbelow(NOTE_SUBGROUP_ORDER - 1) + 1) for _ in range(n)))
        columns = _NOTE_KINDS[kind]
        args = _batch_args(f"{kind}_encrypt", columns, [size * n for _, size, _ in columns], arrays)
        rec, cm, st = C.create_string_buffer(160 * n), C.create_string_buffer(32 * n), C.create_string_buffer(n)
        _check(getattr(lib(), f"og_{kind}_encrypt")(self._h, *args, n, rec, cm, st), self)
        return rec.raw, cm.raw, st.raw[:n]

    def _note_encrypt_dev(self, kind, d_arrays, n, d_outs):
        _check(getattr(lib(), f"og_{kind}_encrypt_dev")(self._h, *[_ptr(x) for x in d_arrays], n, *[_ptr(x) for x in d_outs]), self)

    def _note_scan(self, kind, view_keys, spend_public_keys, records, commitments):
        """og_<kind>_scan -> (owners, plaintexts); spend_public_keys is None for transfer notes."""
        fn = f"{kind}_scan"
        keys = _note_keys(fn, view_keys, spend_public_keys)
        _need(len(records) % 160 == 0, f"{fn}: records must be a multiple of 160 bytes")
        n = len(records) // 160
        _need(len(commitments) == 32 * n, f"{fn}: expected one 32-byte commitment per record")
        owner, plain = (C.c_uint32 * n)(), C.create_string_buffer(128 * n)
        _check(getattr(lib(), f"og_{fn}")(self._h, *keys, records, commitments, n, owner, plain), self)
        return list(owner), plain.raw

    def _note_scan_dev(self, kind, view_keys, spend_public_keys, d_args):
        keys = _note_keys(f"{kind}_scan_dev", view_keys, spend_public_keys)
        d_records, d_commitments, n, d_owner, d_plaintexts = d_args
        _check(getattr(lib(), f"og_{kind}_scan_dev")(self._h, *keys, _ptr(d_records), _ptr(d_commitments), n, _ptr(d_owner),
                                                     _ptr(d_plaintexts)), self)

    # ---- the note hashes: one body for every row of _NOTE_HASHES -----------------------------------------------------
    def _note_hash(self, h, arrays) -> bytes:
        """og_<h> of the items in `arrays` (_NOTE_HASHES[h] order, as many items as the first column has 32-byte elements)
        -> 32 bytes per item."""
        columns = _NOTE_HASHES[h]
        _need(_blen(arrays[0]) is not None and _blen(arrays[0]) % 32 == 0, f"{h}: {columns[0][0]} must be a multiple of 32 bytes")
        n = _blen(arrays[0]) // 32
        args = _batch_args(h, columns, [size * n for _, size, _ in columns], arrays)
        out = C.create_string_buffer(32 * n)
        _check(getattr(lib(), f"og_{h}")(self._h, *args, n, out), self)
        return out.raw

    # ---- encrypted notes (DESIGN.md section 3, "Encrypted notes") ----------------------------------------------------
    def note_public_keys(self, view_keys: bytes):
        """View keys (32 bytes each, canonical, nonzero mod l) -> (pk_x, pk_is_odd): the compressed addresses v BASE."""
        _need(len(view_keys) % 32 == 0, "note_public_keys: view keys must be a multiple of 32 bytes")
        n = len(view_keys) // 32
        px, odd = C.create_string_buffer(32 * n), C.create_string_buffer(n)
        _check(lib().og_note_public_keys(self._h, view_keys, n, px, odd), self)
        return px.raw, odd.raw[:n]

    def note_encrypt(self, pk_x: bytes, pk_is_odd: bytes, nullifiers: bytes, secrets: bytes, tokens: bytes, amounts, ephemerals=None):
        """Encrypt note i to the address (pk_x[i], pk_is_odd[i]) -> (records (160 B each), commitments (32 B each), status)
        with status 1 = written, 2 = the address does not decompress or has 8 V = O, 3 = the ephemeral is 0 mod l.
        Amounts: a sequence of ints < 2^64 or little-endian u64 bytes.  Ephemerals (32 B each) are drawn with the `secrets`
        module in [1, l) when not given; given ones make every byte reproducible."""
        return self._note_encrypt("note", (pk_x, pk_is_odd, nullifiers, secrets, tokens, amounts, ephemerals))

    def note_encrypt_dev(self, d_pk_x, d_pk_is_odd, d_nullifiers, d_secrets, d_tokens, d_amounts, d_ephemerals, n: int,
                         d_out_records, d_out_commitments, d_out_status):
        """og_note_encrypt_dev: device buffers (addresses or tensors), enqueued on the context's stream."""
        self._note_encrypt_dev("note", (d_pk_x, d_pk_is_odd, d_nullifiers, d_secrets, d_tokens, d_amounts, d_ephemerals), n,
                               (d_out_records, d_out_commitments, d_out_status))

    def note_scan(self, view_keys: bytes, records: bytes, commitments: bytes):
        """Trial-decrypt every record under every view key -> (owners, plaintexts): owners[i] is the lowest index of a key
        that owns record i, NOTE_NOT_OWNED or NOTE_MALFORMED; plaintexts holds 128 bytes per record (nullifier, secret, token,
        amount), zero unless owned."""
        return self._note_scan("note", view_keys, None, records, commitments)

    def note_scan_dev(self, view_keys: bytes, d_records, d_commitments, n: int, d_out_owner, d_out_plaintexts):
        """og_note_scan_dev: view keys on the host, every other buffer on the device, enqueued on the context's stream."""
        self._note_scan_dev("note", view_keys, None, (d_records, d_commitments, n, d_out_owner, d_out_plaintexts))

    # ---- spend-key notes (DESIGN.md section 3, "Owned transfers") ---------------------------------------------------
    def owned_note_encrypt(self, pk_x: bytes, pk_is_odd: bytes, owners: bytes, blindings: bytes, tokens: bytes, amounts, ephemerals=None):
        """note_encrypt for spend-key notes (owner P, blinding, token, amount): the same records, with commitments
        MultiMiMC7([P, blinding, token, amount], 4) -> (records, commitments, status)."""
        return self._note_encrypt("owned_note", (pk_x, pk_is_odd, owners, blindings, tokens, amounts, ephemerals))

    def owned_note_encrypt_dev(self, d_pk_x, d_pk_is_odd, d_owners, d_blindings, d_tokens, d_amounts, d_ephemerals, n: int,
                               d_out_records, d_out_commitments, d_out_status):
        """og_owned_note_encrypt_dev: device buffers (addresses or tensors), enqueued on the context's stream."""
        self._note_encrypt_dev("owned_note", (d_pk_x, d_pk_is_odd, d_owners, d_blindings, d_tokens, d_amounts, d_ephemerals), n,
                               (d_out_records, d_out_commitments, d_out_status))

    def owned_note_scan(self, view_keys: bytes, spend_public_keys: bytes, records: bytes, commitments: bytes):
        """note_scan for spend-key notes: key k is (view_keys[k], spend_public_keys[k]) and owns a record only if the record
        decrypts under the view key to a note whose owner is the spend public key and whose key-4 commitment matches ->
        (owners, plaintexts) as note_scan's, the plaintext words being (owner, blinding, token, amount)."""
        return self._note_scan("owned_note", view_keys, spend_public_keys, records, commitments)

    def owned_note_scan_dev(self, view_keys: bytes, spend_public_keys: bytes, d_records, d_commitments, n: int, d_out_owner,
                            d_out_plaintexts):
        """og_owned_note_scan_dev: the keys on the host, every other buffer on the device, enqueued on the context's stream."""
        self._note_scan_dev("owned_note", view_keys, spend_public_keys, (d_records, d_commitments, n, d_out_owner, d_out_plaintexts))

    def owned_public_keys(self, spend_keys: bytes) -> bytes:
        """MultiMiMC7([s], 3) of each spending key (32 bytes each in and out): the owner a sender puts in a note."""
        return self._note_hash("owned_public_keys", (spend_keys,))

    def owned_commitments(self, owners: bytes, blindings: bytes, tokens: bytes, amounts) -> bytes:
        """MultiMiMC7([owner, blinding, token, amount], 4) of each note: owners, blindings, tokens 32 bytes each, amounts
        uint64 (a little-endian buffer, an array or a sequence of ints)."""
        return self._note_hash("owned_commitments", (owners, blindings, tokens, amounts))

    def owned_nullifiers(self, spend_keys: bytes, commitments: bytes, indices) -> bytes:
        """MultiMiMC7([s, commitment, index], 5) of each note at its leaf index (uint32): the nullifier its spend publishes,
        so a wallet sees which of its notes the chain has spent."""
        return self._note_hash("owned_nullifiers", (spend_keys, commitments, indices))

    # ---- owned labeled notes (DESIGN.md section 3, "Owned labeled transfers") ----------------------------------------
    def owned_labeled_precommitments(self, owners: bytes, blindings: bytes) -> bytes:
        """MultiMiMC7([owner, blinding], 6) of each note (32 bytes each in and out): what a depositor sends the node, which
        does not reveal the owner."""
        return self._note_hash("owned_labeled_precommitments", (owners, blindings))

    def owned_labeled_leaves(self, precommitments: bytes, tokens: bytes, amounts, labels) -> bytes:
        """MultiMiMC7([precommitment, token, amount, label], 7) of each note: precommitments and tokens 32 bytes each, amounts
        uint64 and labels uint32 (little-endian buffers, arrays or sequences of ints)."""
        return self._note_hash("owned_labeled_leaves", (precommitments, tokens, amounts, labels))

    def owned_labeled_note_encrypt(self, pk_x: bytes, pk_is_odd: bytes, owners: bytes, blindings: bytes, tokens: bytes, amounts,
                                   labels, ephemerals=None):
        """note_encrypt for owned labeled notes (owner P, blinding, token, amount, label): the records of the four words (P,
        blinding, token, amount + 2^64 label), with the notes' key-7 leaves as commitments -> (records, commitments, status)."""
        return self._note_encrypt("owned_labeled_note", (pk_x, pk_is_odd, owners, blindings, tokens, amounts, labels, ephemerals))

    def owned_labeled_note_encrypt_dev(self, d_pk_x, d_pk_is_odd, d_owners, d_blindings, d_tokens, d_amounts, d_labels, d_ephemerals,
                                       n: int, d_out_records, d_out_commitments, d_out_status):
        """og_owned_labeled_note_encrypt_dev: device buffers (addresses or tensors), enqueued on the context's stream."""
        self._note_encrypt_dev("owned_labeled_note", (d_pk_x, d_pk_is_odd, d_owners, d_blindings, d_tokens, d_amounts, d_labels,
                                                      d_ephemerals), n, (d_out_records, d_out_commitments, d_out_status))

    def owned_labeled_note_scan(self, view_keys: bytes, spend_public_keys: bytes, records: bytes, commitments: bytes):
        """owned_note_scan for owned labeled notes -> (owners, plaintexts, amounts, labels): owners as note_scan's, the
        plaintext words (owner, blinding, token, amount + 2^64 label) as og_owned_labeled_note_scan returns them, and each
        record's amount and label split from word 3 (0 unless owned)."""
        owner, plain = self._note_scan("owned_labeled_note", view_keys, spend_public_keys, records, commitments)
        words3 = [int.from_bytes(plain[128 * i + 96:128 * i + 128], "little") for i in range(len(owner))]
        return owner, plain, [w & ((1 << 64) - 1) for w in words3], [w >> 64 for w in words3]

    def owned_labeled_note_scan_dev(self, view_keys: bytes, spend_public_keys: bytes, d_records, d_commitments, n: int, d_out_owner,
                                    d_out_plaintexts):
        """og_owned_labeled_note_scan_dev: the keys on the host, every other buffer on the device, enqueued on the context's
        stream; the plaintexts keep word 3 = amount + 2^64 label."""
        self._note_scan_dev("owned_labeled_note", view_keys, spend_public_keys, (d_records, d_commitments, n, d_out_owner,
                                                                                 d_out_plaintexts))

    def msm_g1(self, points: bytes, scalars: bytes) -> bytes:
        _need(len(scalars) % 32 == 0, "msm_g1: scalars must be a multiple of 32 bytes")
        n = len(scalars) // 32
        _need(len(points) == 64 * n, "msm_g1: need one 64-byte point per scalar")
        out = C.create_string_buffer(64)
        _check(lib().og_msm_g1(self._h, points, scalars, n, out), self)
        return out.raw

    def msm_g2(self, points: bytes, scalars: bytes) -> bytes:
        _need(len(scalars) % 32 == 0, "msm_g2: scalars must be a multiple of 32 bytes")
        n = len(scalars) // 32
        _need(len(points) == 128 * n, "msm_g2: need one 128-byte point per scalar")
        out = C.create_string_buffer(128)
        _check(lib().og_msm_g2(self._h, points, scalars, n, out), self)
        return out.raw

    def g1_generator_mul(self, scalars: bytes) -> bytes:
        _need(len(scalars) % 32 == 0, "g1_generator_mul: scalars must be a multiple of 32 bytes")
        n = len(scalars) // 32
        out = C.create_string_buffer(64 * n)
        _check(lib().og_g1_generator_mul(self._h, scalars, n, out), self)
        return out.raw

    def g2_generator_mul(self, scalars: bytes) -> bytes:
        _need(len(scalars) % 32 == 0, "g2_generator_mul: scalars must be a multiple of 32 bytes")
        n = len(scalars) // 32
        out = C.create_string_buffer(128 * n)
        _check(lib().og_g2_generator_mul(self._h, scalars, n, out), self)
        return out.raw

    def g1_sum(self, points: bytes) -> bytes:
        _need(len(points) % 64 == 0, "g1_sum: points must be a multiple of 64 bytes")
        out = C.create_string_buffer(64)
        _check(lib().og_g1_sum(self._h, points, len(points) // 64, out), self)
        return out.raw

    def g2_sum(self, points: bytes) -> bytes:
        _need(len(points) % 128 == 0, "g2_sum: points must be a multiple of 128 bytes")
        out = C.create_string_buffer(128)
        _check(lib().og_g2_sum(self._h, points, len(points) // 128, out), self)
        return out.raw

    def ntt(self, data: bytes, log_n: int, batch: int = 1, inverse=False, coset=False) -> bytes:
        _need(0 <= log_n <= 27 and batch >= 0 and len(data) == (32 * batch) << log_n, "ntt: data must hold batch * 2^log_n elements of 32 bytes")
        buf = C.create_string_buffer(data, len(data))
        _check(lib().og_ntt(self._h, buf, log_n, batch, int(inverse), int(coset)), self)
        return buf.raw

    def _statement_witness(self, stmt, depth, arrays) -> bytes:
        """Full assignments of statement `stmt` at `depth`, n_vars * 32 bytes per proof; the batch is the first array's
        32-byte elements."""
        fn, first = f"{stmt}_witness", _STATEMENTS[stmt][1][0][0]
        _need(not _STATEMENTS[stmt][0] or 1 <= depth <= 32, f"{fn}: depth must be 1..32")
        _need(_blen(arrays[0]) is not None and _blen(arrays[0]) % 32 == 0, f"{fn}: {first} must be a multiple of 32 bytes")
        n = _blen(arrays[0]) // 32
        args = _statement_args(stmt, fn, n, depth, arrays)
        out = C.create_string_buffer(32 * n * _statement_r1cs_info(stmt, depth)["n_vars"])
        _check(getattr(lib(), f"og_{stmt}_witness")(self._h, *_depth_arg(stmt, depth), *args, n, out), self)
        return out.raw

    def withdraw_witness(self, depth, nullifiers: bytes, secrets: bytes, recipients: bytes, siblings: bytes, path_bits) -> bytes:
        return self._statement_witness("withdraw", depth, (nullifiers, secrets, recipients, siblings, path_bits))

    def deposit_witness(self, nullifiers: bytes, secrets: bytes, depositors: bytes) -> bytes:
        """Full assignments of the deposit statement, n_vars * 32 bytes per deposit, computed on the GPU."""
        return self._statement_witness("deposit", 0, (nullifiers, secrets, depositors))

    def transfer_witness(self, depth, roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings, in_path_bits,
                         out_nullifiers, out_secrets, out_amounts) -> bytes:
        """Full assignments of the depth-`depth` transfer statement, n_vars * 32 bytes per transfer, computed on the GPU.
        Per transfer: roots / tokens / recipients 32 bytes each; in_* / out_* note 0 then note 1 (nullifiers and secrets
        2 x 32 bytes, amounts 2 x uint64 as 8-byte little-endian buffers, uint64 arrays or ints); in_siblings 2 * depth
        elements (input 0's path, then input 1's); in_path_bits 2 words."""
        return self._statement_witness("transfer", depth, (roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings,
                                                           in_path_bits, out_nullifiers, out_secrets, out_amounts))

    def association_witness(self, depth, nullifiers, secrets, recipients, siblings, path_bits, assoc_siblings, assoc_path_bits) -> bytes:
        """Full assignments of the depth-`depth` association-set withdraw statement, n_vars * 32 bytes per proof, computed on
        the GPU.  Per proof: nullifier, secret, recipient 32 bytes each; siblings and assoc_siblings depth elements each (the
        pool path and the association path, leaf level first); path_bits and assoc_path_bits one word each."""
        return self._statement_witness("association", depth, (nullifiers, secrets, recipients, siblings, path_bits, assoc_siblings,
                                                              assoc_path_bits))

    def exclusion_witness(self, depth, nullifiers, secrets, recipients, siblings, path_bits, excl_low, excl_next, excl_siblings,
                          excl_path_bits) -> bytes:
        """Full assignments of the depth-`depth` exclusion withdraw statement, n_vars * 32 bytes per proof, computed on the
        GPU.  Per proof: nullifier, secret, recipient 32 bytes each; siblings and excl_siblings depth elements each (the pool
        path and the blocklist-tree path, leaf level first); path_bits and excl_path_bits one word each; excl_low and
        excl_next one uint64 each (8-byte little-endian buffers, uint64 arrays or ints), the keys of the blocklist leaf that
        brackets the note (ExclusionSet.witness)."""
        return self._statement_witness("exclusion", depth, (nullifiers, secrets, recipients, siblings, path_bits, excl_low, excl_next,
                                                            excl_siblings, excl_path_bits))

    # ---- labeled notes (DESIGN.md section 3, "Labeled withdrawals") --------------------------------------------------
    def labeled_precommitments(self, nullifiers: bytes, secrets: bytes) -> bytes:
        """MultiMiMC7([nullifier, secret], 2) of each note (32 bytes each in and out): what a depositor sends the node."""
        return self._note_hash("labeled_precommitments", (nullifiers, secrets))

    def labeled_leaves(self, precommitments: bytes, tokens: bytes, amounts, labels) -> bytes:
        """MultiMiMC7([precommitment, token, amount, label], 2) of each deposit: precommitments and tokens 32 bytes each,
        amounts uint64 and labels uint32 (little-endian buffers, arrays or sequences of ints)."""
        return self._note_hash("labeled_leaves", (precommitments, tokens, amounts, labels))

    def labeled_witness(self, depth, tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits,
                        change_nullifiers, change_secrets, excl_low, excl_next, excl_siblings, excl_path_bits) -> bytes:
        """Full assignments of the depth-`depth` labeled withdraw statement, n_vars * 32 bytes per proof, computed on the GPU.
        Per proof: token, recipient, nullifier, secret, change_nullifier, change_secret 32 bytes each; withdrawn, amount,
        excl_low and excl_next one uint64 each and the label one uint32 (little-endian buffers, arrays or ints); siblings
        and excl_siblings depth elements each (the note's pool path and the blocklist-tree path of its label,
        ExclusionSet.witness), path_bits and excl_path_bits one word each."""
        return self._statement_witness("labeled", depth, (tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings,
                                                          path_bits, change_nullifiers, change_secrets, excl_low, excl_next,
                                                          excl_siblings, excl_path_bits))

    def labeled_association_witness(self, depth, tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings,
                                    path_bits, change_nullifiers, change_secrets, assoc_siblings, assoc_path_bits) -> bytes:
        """Full assignments of the depth-`depth` labeled association withdraw statement, n_vars * 32 bytes per proof, computed
        on the GPU.  The first eleven inputs as in labeled_witness; assoc_siblings depth elements and assoc_path_bits one word
        per proof (the path of the label's leaf in the provider's tree, ApprovedLabels.witness)."""
        return self._statement_witness("labeled_association", depth, (tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels,
                                                                      siblings, path_bits, change_nullifiers, change_secrets,
                                                                      assoc_siblings, assoc_path_bits))

    def owned_transfer_witness(self, depth, roots, tokens, recipients, in_spend_keys, in_blindings, in_amounts, in_siblings,
                               in_path_bits, out_owners, out_blindings, out_amounts) -> bytes:
        """Full assignments of the depth-`depth` owned transfer statement, n_vars * 32 bytes per transfer, computed on the GPU.
        Inputs as in transfer_witness, with the inputs' spending keys and blindings in place of their nullifiers and secrets
        and the outputs' owners (spend public keys) and blindings in place of theirs."""
        return self._statement_witness("owned_transfer", depth, (roots, tokens, recipients, in_spend_keys, in_blindings, in_amounts,
                                                                 in_siblings, in_path_bits, out_owners, out_blindings, out_amounts))

    def owned_labeled_transfer_witness(self, depth, roots, tokens, recipients, withdrawn, labels, in_spend_keys, in_blindings,
                                       in_amounts, in_siblings, in_path_bits, out_owners, out_blindings, out_amounts, assoc_siblings,
                                       assoc_path_bits) -> bytes:
        """Full assignments of the depth-`depth` owned labeled transfer statement, n_vars * 32 bytes per transfer, computed on
        the GPU.  Per transfer: root, token, recipient 32 bytes each; withdrawn one uint64 and the label one uint32; the inputs
        and outputs as in owned_transfer_witness; assoc_siblings depth elements and assoc_path_bits one word, the path of
        label + 1 in the provider's approved-label tree (ApprovedLabels.witness)."""
        return self._statement_witness("owned_labeled_transfer", depth, (roots, tokens, recipients, withdrawn, labels, in_spend_keys,
                                                                         in_blindings, in_amounts, in_siblings, in_path_bits, out_owners,
                                                                         out_blindings, out_amounts, assoc_siblings, assoc_path_bits))

    def ragequit_witness(self, depth, roots, tokens, recipients, amounts, labels, spend_keys, blindings, siblings, path_bits) -> bytes:
        """Full assignments of the depth-`depth` ragequit statement, n_vars * 32 bytes per proof, computed on the GPU.  Per
        proof: root, token, recipient 32 bytes each; the note's amount one uint64 and its label one uint32; its spending key
        and blinding 32 bytes each; siblings depth elements and path_bits one word, the note's pool path."""
        return self._statement_witness("ragequit", depth, (roots, tokens, recipients, amounts, labels, spend_keys, blindings, siblings,
                                                           path_bits))


def mimc7_constants():
    out = C.create_string_buffer(32 * 91)
    n = C.c_uint32()
    _check(lib().og_mimc7_constants(out, C.byref(n)))
    return [int.from_bytes(out.raw[32 * i:32 * i + 32], "little") for i in range(n.value)]


def _statement_r1cs_info(stmt, depth) -> dict:
    v = [C.c_uint32() for _ in range(4)]
    _check(getattr(lib(), f"og_{stmt}_r1cs_info")(*_depth_arg(stmt, depth), *[C.byref(x) for x in v]))
    return dict(n_constraints=v[0].value, n_vars=v[1].value, n_pub=v[2].value, log_m=v[3].value)


def _statement_r1cs_export(stmt, depth, which):
    w = "ABC".index(which)
    export = getattr(lib(), f"og_{stmt}_r1cs_export")
    nnz = C.c_uint64()
    _check(export(*_depth_arg(stmt, depth), w, None, None, None, C.byref(nnz)))
    nc = _statement_r1cs_info(stmt, depth)["n_constraints"]
    ptr = (C.c_uint32 * (nc + 1))()
    col = (C.c_uint32 * nnz.value)()
    val = C.create_string_buffer(32 * nnz.value)
    _check(export(*_depth_arg(stmt, depth), w, ptr, col, val, C.byref(nnz)))
    return list(ptr), list(col), [int.from_bytes(val.raw[32 * i:32 * i + 32], "little") for i in range(nnz.value)]


def r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("withdraw", depth)


def r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's withdraw R1CS."""
    return _statement_r1cs_export("withdraw", depth, which)


def deposit_r1cs_info() -> dict:
    return _statement_r1cs_info("deposit", 0)


def deposit_r1cs_export(which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's deposit R1CS."""
    return _statement_r1cs_export("deposit", 0, which)


def transfer_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("transfer", depth)


def transfer_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` transfer R1CS."""
    return _statement_r1cs_export("transfer", depth, which)


def association_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("association", depth)


def association_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` association R1CS."""
    return _statement_r1cs_export("association", depth, which)


def exclusion_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("exclusion", depth)


def exclusion_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` exclusion R1CS."""
    return _statement_r1cs_export("exclusion", depth, which)


def labeled_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("labeled", depth)


def labeled_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` labeled withdraw R1CS."""
    return _statement_r1cs_export("labeled", depth, which)


def labeled_association_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("labeled_association", depth)


def labeled_association_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` labeled association R1CS."""
    return _statement_r1cs_export("labeled_association", depth, which)


def owned_transfer_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("owned_transfer", depth)


def owned_transfer_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` owned transfer R1CS."""
    return _statement_r1cs_export("owned_transfer", depth, which)


def owned_labeled_transfer_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("owned_labeled_transfer", depth)


def owned_labeled_transfer_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` owned labeled transfer R1CS."""
    return _statement_r1cs_export("owned_labeled_transfer", depth, which)


def ragequit_r1cs_info(depth: int) -> dict:
    return _statement_r1cs_info("ragequit", depth)


def ragequit_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` ragequit R1CS."""
    return _statement_r1cs_export("ragequit", depth, which)


def _r1cs_args(A, B, C_):
    """(n_constraints, the nine CSR arguments of og_groth16_setup / og_ptau_prepare) after the length checks."""
    mats = []
    n_constraints = None
    for name, M in (("A", A), ("B", B), ("C", C_)):
        _need(len(M) == 3, f"setup_r1cs: {name} must be a (row_ptr, col_idx, coeffs) triple")
        ptr, col, val = M
        _need(len(ptr) >= 2, f"setup_r1cs: {name}.row_ptr needs n_constraints + 1 >= 2 entries")
        _need(n_constraints is None or len(ptr) == n_constraints + 1, f"setup_r1cs: {name}.row_ptr length differs from A's")
        n_constraints = len(ptr) - 1
        _need(len(col) == len(val), f"setup_r1cs: {name}.col_idx and {name}.coeffs differ in length")
        _need(ptr[-1] == len(col), f"setup_r1cs: {name}.row_ptr ends at {ptr[-1]}, but there are {len(col)} terms")
        _need(all(0 <= x < 1 << 32 for x in ptr) and all(0 <= x < 1 << 32 for x in col), f"setup_r1cs: {name} indices must be 32-bit")
        cb = b"".join(bytes(x) if isinstance(x, (bytes, bytearray)) else int(x).to_bytes(32, "little") for x in val)
        _need(len(cb) == 32 * len(val), f"setup_r1cs: {name} coefficients are 32 bytes each")
        mats += [(C.c_uint32 * len(ptr))(*ptr), (C.c_uint32 * max(1, len(col)))(*col), cb]
    return n_constraints, mats


def setup_r1cs(ctx: Context, n_vars: int, n_pub: int, A, B, C_, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of any R1CS -> (pk_bytes, vk_bytes).  A, B, C_ are (row_ptr, col_idx, coeffs) triples as
    r1cs_export returns them (coefficients as ints or 32-byte little-endian values); variable 0 is ONE and variables
    1..n_pub are the public inputs.  The key records depth 0, so it proves through prove_witnesses."""
    n_constraints, mats = _r1cs_args(A, B, C_)
    toxic = b"".join(fr_bytes(x) for x in (tau, alpha, beta, gamma, delta))
    pl, vl = C.c_uint64(), C.c_uint64()
    _check(lib().og_groth16_setup(ctx._h, n_constraints, n_vars, n_pub, *mats, toxic, None, C.byref(pl), None, C.byref(vl)), ctx)
    pk = C.create_string_buffer(pl.value)
    vk = C.create_string_buffer(vl.value)
    _check(lib().og_groth16_setup(ctx._h, n_constraints, n_vars, n_pub, *mats, toxic, pk, C.byref(pl), vk, C.byref(vl)), ctx)
    return pk.raw[:pl.value], vk.raw[:vl.value]


def _setup_statement(ctx, stmt, depth, toxic):
    info = _statement_r1cs_info(stmt, depth)
    return setup_r1cs(ctx, info["n_vars"], info["n_pub"], *(_statement_r1cs_export(stmt, depth, m) for m in "ABC"), *toxic)


def setup_deposit(ctx: Context, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the deposit statement -> (pk_bytes, vk_bytes): its exported R1CS through setup_r1cs."""
    return _setup_statement(ctx, "deposit", 0, (tau, alpha, beta, gamma, delta))


def setup_transfer(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` transfer statement -> (pk_bytes, vk_bytes): its exported R1CS through
    setup_r1cs.  The key records depth 0; the prover recognises it as a transfer key by its shape."""
    return _setup_statement(ctx, "transfer", depth, (tau, alpha, beta, gamma, delta))


def setup_association(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` association-set withdraw statement -> (pk_bytes, vk_bytes): its exported R1CS
    through setup_r1cs.  The key records depth 0; the prover recognises it as an association key by its shape."""
    return _setup_statement(ctx, "association", depth, (tau, alpha, beta, gamma, delta))


def setup_exclusion(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` exclusion withdraw statement -> (pk_bytes, vk_bytes): its exported R1CS through
    setup_r1cs.  The key records depth 0; the prover recognises it as an exclusion key by its shape."""
    return _setup_statement(ctx, "exclusion", depth, (tau, alpha, beta, gamma, delta))


def setup_labeled(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` labeled withdraw statement -> (pk_bytes, vk_bytes): its exported R1CS through
    setup_r1cs.  The key records depth 0; the prover recognises it as a labeled key by its shape."""
    return _setup_statement(ctx, "labeled", depth, (tau, alpha, beta, gamma, delta))


def setup_labeled_association(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` labeled association withdraw statement -> (pk_bytes, vk_bytes): its exported
    R1CS through setup_r1cs.  The key records depth 0; the prover recognises it as a labeled association key by its shape."""
    return _setup_statement(ctx, "labeled_association", depth, (tau, alpha, beta, gamma, delta))


def setup_owned_transfer(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` owned transfer statement -> (pk_bytes, vk_bytes): its exported R1CS through
    setup_r1cs.  The key records depth 0; the prover recognises it as an owned transfer key by its shape."""
    return _setup_statement(ctx, "owned_transfer", depth, (tau, alpha, beta, gamma, delta))


def setup_owned_labeled_transfer(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` owned labeled transfer statement -> (pk_bytes, vk_bytes): its exported R1CS
    through setup_r1cs.  The key records depth 0; the prover recognises it as an owned labeled transfer key by its shape."""
    return _setup_statement(ctx, "owned_labeled_transfer", depth, (tau, alpha, beta, gamma, delta))


def setup_ragequit(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` ragequit statement -> (pk_bytes, vk_bytes): its exported R1CS through
    setup_r1cs.  The key records depth 0; the prover recognises it as a ragequit key by its shape."""
    return _setup_statement(ctx, "ragequit", depth, (tau, alpha, beta, gamma, delta))


def setup_withdraw(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup (toxic waste supplied by the caller) -> (pk_bytes, vk_bytes)."""
    toxic = b"".join(fr_bytes(x) for x in (tau, alpha, beta, gamma, delta))
    pl, vl = C.c_uint64(), C.c_uint64()
    _check(lib().og_groth16_setup_withdraw(ctx._h, depth, toxic, None, C.byref(pl), None, C.byref(vl)), ctx)
    pk = C.create_string_buffer(pl.value)
    vk = C.create_string_buffer(vl.value)
    _check(lib().og_groth16_setup_withdraw(ctx._h, depth, toxic, pk, C.byref(pl), vk, C.byref(vl)), ctx)
    return pk.raw[:pl.value], vk.raw[:vl.value]


# ---- two-phase setup ceremony (DESIGN.md section 4b) -------------------------------------------------------------------
def _sized(ctx, fn, n_out=1):
    """Call fn(*out_args) twice (NULL -> sizes, then the buffers) and return its n_out blobs."""
    lens = [C.c_uint64() for _ in range(n_out)]
    _check(fn(*[a for x in lens for a in (None, C.byref(x))]), ctx)
    bufs = [C.create_string_buffer(x.value) for x in lens]
    _check(fn(*[a for b, x in zip(bufs, lens) for a in (b, C.byref(x))]), ctx)
    out = [b.raw[:x.value] for b, x in zip(bufs, lens)]
    return out[0] if n_out == 1 else tuple(out)


def _secrets(xs, n, name):
    if xs is None:
        return [_rand.randbelow(FR_MODULUS - 1) + 1 for _ in range(n)]
    xs = list(xs)
    _need(len(xs) == n, f"{name}: expected {n} values")
    return xs


def ptau_new(ctx: Context, log_max: int) -> bytes:
    """The initial powers-of-tau accumulator of size M = 2^log_max (every point a generator)."""
    return _sized(ctx, lambda *io: lib().og_ptau_new(ctx._h, log_max, *io))


def ptau_contribute(ctx: Context, acc: bytes, secrets=None, nonces=None):
    """Apply secrets (t, a, b) to an accumulator -> (new accumulator, record).  Secrets and nonces are drawn with the
    `secrets` module when not given; given ones make every byte reproducible."""
    s = _secrets(secrets, 3, "ptau_contribute: secrets")
    k = _secrets(nonces, 3, "ptau_contribute: nonces")
    sb, kb = b"".join(fr_bytes(x) for x in s), b"".join(fr_bytes(x) for x in k)
    return _sized(ctx, lambda *io: lib().og_ptau_contribute(ctx._h, acc, len(acc), sb, kb, *io), n_out=2)


def ptau_verify(ctx: Context, prev: bytes, nxt: bytes, record: bytes) -> bool:
    """True iff `nxt` is `prev` updated by the contribution that `record` proves knowledge of."""
    rc = lib().og_ptau_verify(ctx._h, prev, len(prev), nxt, len(nxt), record, len(record))
    if rc in (OG_OK, OG_E_VERIFY):
        return rc == OG_OK
    _check(rc, ctx)


def ptau_prepare(ctx: Context, acc: bytes, n_vars: int, n_pub: int, A, B, C_):
    """The phase-2 starting key (pk, vk) of any R1CS from an accumulator: arguments as setup_r1cs; the key records depth 0."""
    n_constraints, mats = _r1cs_args(A, B, C_)
    return _sized(ctx, lambda *io: lib().og_ptau_prepare(ctx._h, acc, len(acc), n_constraints, n_vars, n_pub, *mats, *io), n_out=2)


def ptau_prepare_withdraw(ctx: Context, acc: bytes, depth: int):
    """The phase-2 starting key of the depth-`depth` withdraw statement (the depth is recorded, as setup_withdraw)."""
    return _sized(ctx, lambda *io: lib().og_ptau_prepare_withdraw(ctx._h, acc, len(acc), depth, *io), n_out=2)


def _ptau_prepare_statement(ctx, acc, stmt, depth):
    info = _statement_r1cs_info(stmt, depth)
    return ptau_prepare(ctx, acc, info["n_vars"], info["n_pub"], *(_statement_r1cs_export(stmt, depth, m) for m in "ABC"))


def ptau_prepare_deposit(ctx: Context, acc: bytes):
    return _ptau_prepare_statement(ctx, acc, "deposit", 0)


def ptau_prepare_transfer(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "transfer", depth)


def ptau_prepare_association(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "association", depth)


def ptau_prepare_exclusion(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "exclusion", depth)


def ptau_prepare_labeled(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "labeled", depth)


def ptau_prepare_labeled_association(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "labeled_association", depth)


def ptau_prepare_owned_transfer(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "owned_transfer", depth)


def ptau_prepare_owned_labeled_transfer(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "owned_labeled_transfer", depth)


def ptau_prepare_ragequit(ctx: Context, acc: bytes, depth: int):
    return _ptau_prepare_statement(ctx, acc, "ragequit", depth)


def phase2_contribute(ctx: Context, pk: bytes, vk: bytes, delta=None, nonce=None):
    """Multiply the key's delta by a secret d -> (pk, vk, record); d and the nonce are drawn with `secrets` when not given."""
    d = _secrets(None if delta is None else [delta], 1, "phase2_contribute: delta")[0]
    k = _secrets(None if nonce is None else [nonce], 1, "phase2_contribute: nonce")[0]
    return _sized(ctx, lambda *io: lib().og_phase2_contribute(ctx._h, pk, len(pk), vk, len(vk), fr_bytes(d), fr_bytes(k), *io),
                  n_out=3)


def phase2_verify(ctx: Context, pk_prev: bytes, vk_prev: bytes, pk_next: bytes, vk_next: bytes, record: bytes) -> bool:
    rc = lib().og_phase2_verify(ctx._h, pk_prev, len(pk_prev), vk_prev, len(vk_prev), pk_next, len(pk_next), vk_next, len(vk_next),
                                record, len(record))
    if rc in (OG_OK, OG_E_VERIFY):
        return rc == OG_OK
    _check(rc, ctx)


class ProvingKey:
    """A proving key resident in HBM together with its fixed-base window tables (og_pk)."""

    def __init__(self, ctx: Context, pk_bytes: bytes):
        self.ctx = ctx
        self._h = C.c_void_p()
        _check(lib().og_load_pk(ctx._h, pk_bytes, len(pk_bytes), C.byref(self._h)), ctx)
        v = [C.c_uint32() for _ in range(4)]
        _check(lib().og_pk_info(self._h, *[C.byref(x) for x in v]))
        self.n_vars, self.n_pub, self.log_m, self.depth = (x.value for x in v)

    def close(self):
        # always release the device tables: the key records its device itself and may outlive its Context
        if getattr(self, "_h", None) and _lib is not None:
            _lib.og_free_pk(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def window_bits(self):
        """(A, B, C') window bits of the prover's three MSMs for this key."""
        c = (C.c_uint32 * 3)()
        _check(lib().og_pk_window_bits(self._h, c))
        return tuple(c)

    def h_evals(self, witness: bytes) -> bytes:
        _need(len(witness) == 32 * self.n_vars, f"h_evals: a witness is {32 * self.n_vars} bytes")
        out = C.create_string_buffer(32 << self.log_m)
        _check(lib().og_groth16_h_evals(self.ctx._h, self._h, witness, out), self.ctx)
        return out.raw

    def prove_witnesses(self, witnesses: bytes, rs: bytes) -> bytes:
        _need(len(rs) % 64 == 0, "prove_witnesses: rs holds 64 bytes (r, s) per proof")
        batch = len(rs) // 64
        _need(len(witnesses) == 32 * batch * self.n_vars, f"prove_witnesses: need {32 * self.n_vars} witness bytes per proof")
        out = C.create_string_buffer(PROOF_BYTES * batch)
        _check(lib().og_groth16_prove(self.ctx._h, self._h, witnesses, batch, rs, out), self.ctx)
        return out.raw

    def _prove_statement(self, stmt, depth, arrays, rs, want_public, batch=None):
        """Proofs of statement `stmt` at `depth` (None: the key is not the statement's); the batch is rs's 64-byte (r, s)
        pairs unless given."""
        fn = f"prove_{stmt}"
        if depth is None:
            raise OwshenB200Error(OG_E_INVALID, f"{fn}: this key was not made for the {stmt} statement")
        if batch is None:
            _need(_blen(rs) is not None and _blen(rs) % 64 == 0, f"{fn}: rs must be a buffer of 64 bytes (r, s) per proof")
            batch = _blen(rs) // 64
        args = _statement_args(stmt, fn, batch, depth, arrays)
        _need_len(rs, 64 * batch, f"{fn}: rs")
        proofs = C.create_string_buffer(PROOF_BYTES * batch)
        pub = C.create_string_buffer(32 * self.n_pub * batch) if want_public else None
        _check(getattr(lib(), f"og_groth16_prove_{stmt}")(self.ctx._h, self._h, *args, batch, _ptr(rs), proofs, pub), self.ctx)
        return proofs.raw, (pub.raw if want_public else None)

    def _shape_depth(self, stmt):
        """The depth d in 1..32 whose statement `stmt` has this key's shape (n_vars, n_pub), or None."""
        for d in range(1, 33):
            info = _statement_r1cs_info(stmt, d)
            if (info["n_vars"], info["n_pub"]) == (self.n_vars, self.n_pub):
                return d
        return None

    def prove_withdraw(self, nullifiers, secrets, recipients, siblings, path_bits, rs, want_public=True):
        """Host buffers in, host buffers out (H2D / D2H inside).  Buffers may be bytes or pinned
        tensors / arrays exposing data_ptr() / .ctypes.  Returns (proofs, public_inputs)."""
        _need(self.depth >= 1, "prove_withdraw: this key was not made for the withdraw statement")
        return self._prove_statement("withdraw", self.depth, (nullifiers, secrets, recipients, siblings, path_bits), rs, want_public,
                                     batch=len(path_bits))

    def prove_deposit(self, nullifiers, secrets, depositors, rs, want_public=True):
        """Batch of deposit proofs from the secret inputs (witness generation on the GPU).  Buffers as in prove_withdraw;
        returns (proofs, public_inputs) with public inputs (commitment, depositor) per proof."""
        return self._prove_statement("deposit", 0, (nullifiers, secrets, depositors), rs, want_public)

    @property
    def transfer_depth(self):
        """The depth d whose transfer statement has this key's shape (transfer_r1cs_info), or None."""
        return self._shape_depth("transfer")

    def prove_transfer(self, roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings, in_path_bits,
                       out_nullifiers, out_secrets, out_amounts, rs, want_public=True):
        """Batch of transfer proofs from the notes (witness generation on the GPU).  Inputs as in Context.transfer_witness;
        returns (proofs, public_inputs) with public inputs (root, public_amount, token, recipient, nullifier_hash[2],
        out_commitment[2]) per proof."""
        return self._prove_statement("transfer", self.transfer_depth, (roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts,
                                                                       in_siblings, in_path_bits, out_nullifiers, out_secrets,
                                                                       out_amounts), rs, want_public)

    @property
    def association_depth(self):
        """The depth d whose association statement has this key's shape (association_r1cs_info), or None."""
        return self._shape_depth("association")

    def prove_association(self, nullifiers, secrets, recipients, siblings, path_bits, assoc_siblings, assoc_path_bits, rs,
                          want_public=True):
        """Batch of association-set withdraw proofs from the secret inputs (witness generation on the GPU).  Inputs as in
        Context.association_witness; returns (proofs, public_inputs) with public inputs (root, nullifier_hash, recipient,
        association_root) per proof."""
        return self._prove_statement("association", self.association_depth,
                                     (nullifiers, secrets, recipients, siblings, path_bits, assoc_siblings, assoc_path_bits), rs, want_public)

    @property
    def exclusion_depth(self):
        """The depth d whose exclusion statement has this key's shape (exclusion_r1cs_info), or None."""
        return self._shape_depth("exclusion")

    def prove_exclusion(self, nullifiers, secrets, recipients, siblings, path_bits, excl_low, excl_next, excl_siblings, excl_path_bits,
                        rs, want_public=True):
        """Batch of exclusion withdraw proofs from the secret inputs (witness generation on the GPU).  Inputs as in
        Context.exclusion_witness; returns (proofs, public_inputs) with public inputs (root, nullifier_hash, recipient,
        exclusion_root) per proof."""
        return self._prove_statement("exclusion", self.exclusion_depth,
                                     (nullifiers, secrets, recipients, siblings, path_bits, excl_low, excl_next, excl_siblings,
                                      excl_path_bits), rs, want_public)

    @property
    def labeled_depth(self):
        """The depth d whose labeled statement has this key's shape (labeled_r1cs_info), or None."""
        return self._shape_depth("labeled")

    def prove_labeled(self, tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits, change_nullifiers,
                      change_secrets, excl_low, excl_next, excl_siblings, excl_path_bits, rs, want_public=True):
        """Batch of labeled withdraw proofs from the notes (witness generation on the GPU).  Inputs as in
        Context.labeled_witness; returns (proofs, public_inputs) with public inputs (root, nullifier_hash, recipient,
        exclusion_root, token, withdrawn, change_commitment) per proof."""
        return self._prove_statement("labeled", self.labeled_depth,
                                     (tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits,
                                      change_nullifiers, change_secrets, excl_low, excl_next, excl_siblings, excl_path_bits), rs,
                                     want_public)

    @property
    def labeled_association_depth(self):
        """The depth d whose labeled association statement has this key's shape (labeled_association_r1cs_info), or None."""
        return self._shape_depth("labeled_association")

    def prove_labeled_association(self, tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits,
                                  change_nullifiers, change_secrets, assoc_siblings, assoc_path_bits, rs, want_public=True):
        """Batch of labeled association withdraw proofs from the notes (witness generation on the GPU).  Inputs as in
        Context.labeled_association_witness; returns (proofs, public_inputs) with public inputs (root, nullifier_hash,
        recipient, association_root, token, withdrawn, change_commitment) per proof."""
        return self._prove_statement("labeled_association", self.labeled_association_depth,
                                     (tokens, recipients, withdrawn, nullifiers, secrets, amounts, labels, siblings, path_bits,
                                      change_nullifiers, change_secrets, assoc_siblings, assoc_path_bits), rs, want_public)

    @property
    def owned_transfer_depth(self):
        """The depth d whose owned transfer statement has this key's shape (owned_transfer_r1cs_info), or None."""
        return self._shape_depth("owned_transfer")

    def prove_owned_transfer(self, roots, tokens, recipients, in_spend_keys, in_blindings, in_amounts, in_siblings, in_path_bits,
                             out_owners, out_blindings, out_amounts, rs, want_public=True):
        """Batch of owned transfer proofs from the notes (witness generation on the GPU).  Inputs as in
        Context.owned_transfer_witness; returns (proofs, public_inputs) with public inputs (root, public_amount, token,
        recipient, nullifier[2], out_commitment[2]) per proof."""
        return self._prove_statement("owned_transfer", self.owned_transfer_depth,
                                     (roots, tokens, recipients, in_spend_keys, in_blindings, in_amounts, in_siblings, in_path_bits,
                                      out_owners, out_blindings, out_amounts), rs, want_public)

    @property
    def owned_labeled_transfer_depth(self):
        """The depth d whose owned labeled transfer statement has this key's shape (owned_labeled_transfer_r1cs_info), or
        None."""
        return self._shape_depth("owned_labeled_transfer")

    def prove_owned_labeled_transfer(self, roots, tokens, recipients, withdrawn, labels, in_spend_keys, in_blindings, in_amounts,
                                     in_siblings, in_path_bits, out_owners, out_blindings, out_amounts, assoc_siblings, assoc_path_bits,
                                     rs, want_public=True):
        """Batch of owned labeled transfer proofs from the notes (witness generation on the GPU).  Inputs as in
        Context.owned_labeled_transfer_witness; returns (proofs, public_inputs) with public inputs (root, association_root,
        token, withdrawn, recipient, nullifier[2], out_commitment[2]) per proof."""
        return self._prove_statement("owned_labeled_transfer", self.owned_labeled_transfer_depth,
                                     (roots, tokens, recipients, withdrawn, labels, in_spend_keys, in_blindings, in_amounts, in_siblings,
                                      in_path_bits, out_owners, out_blindings, out_amounts, assoc_siblings, assoc_path_bits), rs,
                                     want_public)

    @property
    def ragequit_depth(self):
        """The depth d whose ragequit statement has this key's shape (ragequit_r1cs_info), or None."""
        return self._shape_depth("ragequit")

    def prove_ragequit(self, roots, tokens, recipients, amounts, labels, spend_keys, blindings, siblings, path_bits, rs,
                       want_public=True):
        """Batch of ragequit proofs from the notes (witness generation on the GPU).  Inputs as in Context.ragequit_witness;
        returns (proofs, public_inputs) with public inputs (root, token, amount, label, recipient, nullifier) per proof."""
        return self._prove_statement("ragequit", self.ragequit_depth,
                                     (roots, tokens, recipients, amounts, labels, spend_keys, blindings, siblings, path_bits), rs,
                                     want_public)

    def prover_plan(self, batch: int) -> dict:
        """How the prover runs `batch` proofs with this key: chunk (proofs per chunk), lanes (chunks in flight) and
        scratch_bytes_per_lane.  OG_CHUNK / OG_LANES in the environment override the defaults."""
        c, l, s = C.c_uint32(), C.c_uint32(), C.c_uint64()
        _check(lib().og_pk_prover_plan(self._h, batch, C.byref(c), C.byref(l), C.byref(s)))
        return dict(chunk=c.value, lanes=l.value, scratch_bytes_per_lane=s.value)


def prove(pk: ProvingKey, nullifiers, secrets, recipients, siblings, path_bits, rs):
    """prove(): batch of withdraw proofs from the secret inputs -> (proofs bytes, public inputs bytes)."""
    return pk.prove_withdraw(nullifiers, secrets, recipients, siblings, path_bits, rs)


def verify(vk_bytes: bytes, public_inputs: bytes, proof: bytes) -> bool:
    """verify(): True / False for well-formed input, raises OwshenB200Error on malformed encodings."""
    _need(len(proof) == PROOF_BYTES, f"verify: a proof is {PROOF_BYTES} bytes")
    _need(len(public_inputs) % 32 == 0, "verify: public inputs are 32-byte field elements")
    _need(len(vk_bytes) >= 12, "verify: verifying key too short")
    n_pub = len(public_inputs) // 32
    rc = lib().og_groth16_verify(vk_bytes, len(vk_bytes), public_inputs, n_pub, proof)
    if rc == OG_OK:
        return True
    if rc == OG_E_VERIFY:
        return False
    raise OwshenB200Error(rc)


class MerkleTree:
    """Fixed-depth sparse MiMC7 Merkle tree; every hash runs in the CUDA library, nodes live behind a
    KvStore-shaped interface (owshen_b200/kvstore.py, mirroring /root/reference/src/db/mod.rs:24-52), so a tree
    can be reopened over the same store.

    insert_batch() appends leaves: ONE library call (og_mimc7_merkle_append) hashes every touched ancestor on the
    GPU -- the only stored values it needs are the <= depth left-boundary nodes -- and one batch_put commits the
    nodes together with the undo record of the batch, the way the reference commits a block together with its
    `Key::Delta` (src/blockchain/mod.rs:283-286).  pop_batch() applies the newest undo record like `pop_block`
    (src/blockchain/mod.rs:291-315); rollback(n) pops / re-inserts until exactly n leaves remain.
    path(i) returns (siblings bytes, path_bits int)."""

    def __init__(self, ctx: Context, depth: int, store=None, prefix: bytes = b"mt/"):
        from .kvstore import RamKvStore
        _need(1 <= depth <= 32, "MerkleTree: depth must be in 1..32")
        self.ctx, self.depth = ctx, depth
        self.store = store if store is not None else RamKvStore()
        self.prefix = prefix
        self.zeros = [bytes(32)]
        for _ in range(depth):
            self.zeros.append(ctx.mimc7_hash2(self.zeros[-1], self.zeros[-1]))
        d = self.store.get_raw(prefix + b"depth")
        if d is not None and int.from_bytes(d, "little") != depth:
            raise ValueError("store holds a tree of a different depth")

    # ---- state kept in the store (so that a reopened tree sees it) ----------------------------------------
    @property
    def n_leaves(self) -> int:
        n = self.store.get_raw(self.prefix + b"n")
        return int.from_bytes(n, "little") if n else 0

    @property
    def n_batches(self) -> int:
        n = self.store.get_raw(self.prefix + b"height")
        return int.from_bytes(n, "little") if n else 0

    def _key(self, lvl: int, idx: int) -> bytes:
        return self.prefix + lvl.to_bytes(1, "little") + idx.to_bytes(8, "little")

    def _delta_key(self, height: int) -> bytes:
        return self.prefix + b"delta" + height.to_bytes(8, "little")

    def _get(self, lvl, idx):
        v = self.store.get_raw(self._key(lvl, idx))
        return v if v is not None else self.zeros[lvl]

    @staticmethod
    def _pack_delta(delta) -> bytes:
        out = bytearray()
        for k, v in sorted(delta.items()):
            out += len(k).to_bytes(2, "little") + k
            out += b"\x00" if v is None else b"\x01" + len(v).to_bytes(4, "little") + v
        return bytes(out)

    @staticmethod
    def _unpack_delta(blob: bytes):
        out, o = [], 0
        while o < len(blob):
            kl = int.from_bytes(blob[o:o + 2], "little"); o += 2
            k = blob[o:o + kl]; o += kl
            tag = blob[o]; o += 1
            if tag == 0:
                out.append((k, None))
            else:
                vl = int.from_bytes(blob[o:o + 4], "little"); o += 4
                out.append((k, blob[o:o + vl])); o += vl
        return out

    def insert_batch(self, leaves):
        from .kvstore import MirrorKvStore
        leaves = [bytes(x) if isinstance(x, (bytes, bytearray)) else fr_bytes(x) for x in leaves]
        n, start = len(leaves), self.n_leaves
        if n == 0:
            return []
        _need(all(len(x) == 32 for x in leaves), "insert_batch: a leaf is 32 bytes")
        if start + n > (1 << self.depth):
            raise OverflowError(f"tree of depth {self.depth} holds {1 << self.depth} leaves; {start} present, {n} more requested")
        # the only stored nodes the new hashes depend on: (l, (start >> l) - 1) where (start >> l) is odd
        boundary = b"".join(self._get(l, (start >> l) - 1) if (start >> l) & 1 else bytes(32) for l in range(self.depth))
        counts = [((start + n - 1) >> l) - (start >> l) + 1 for l in range(1, self.depth + 1)]
        nodes = self.ctx.merkle_append(self.depth, start, b"".join(leaves), boundary, b"".join(self.zeros[:self.depth]))
        _need(len(nodes) == 32 * sum(counts), "merkle_append returned the wrong number of nodes")
        overlay = MirrorKvStore(self.store)
        overlay.batch_put_raw((self._key(0, start + k), leaf) for k, leaf in enumerate(leaves))
        o = 0
        for l, cnt in zip(range(1, self.depth + 1), counts):
            first = start >> l
            overlay.batch_put_raw((self._key(l, first + k), nodes[o + 32 * k:o + 32 * k + 32]) for k in range(cnt))
            o += 32 * cnt
        height = self.n_batches
        overlay.batch_put_raw([(self.prefix + b"n", (start + n).to_bytes(8, "little")),
                               (self.prefix + b"depth", self.depth.to_bytes(1, "little")),
                               (self.prefix + b"height", (height + 1).to_bytes(8, "little"))])
        delta = overlay.rollback()                       # old value of every key this batch overwrites
        overlay.batch_put_raw([(self._delta_key(height + 1), self._pack_delta(delta))])
        self.store.batch_put_raw(overlay.buffer().items())
        return list(range(start, start + n))

    def insert(self, leaf) -> int:
        return self.insert_batch([leaf])[0]

    def pop_batch(self) -> int:
        """Undo the newest insert_batch (the tree's `pop_block`); returns how many leaves it removed."""
        height = self.n_batches
        if height == 0:
            return 0
        blob = self.store.get_raw(self._delta_key(height))
        if blob is None:
            raise KeyError("Delta not found!")            # the reference's wording, src/blockchain/mod.rs:305
        before = self.n_leaves
        self.store.batch_put_raw(self._unpack_delta(blob) + [(self._delta_key(height), None)])
        return before - self.n_leaves

    def rollback(self, n_leaves: int) -> None:
        """Shrink the tree to exactly n_leaves leaves: whole batches are popped; when the target falls inside a
        batch, that batch is popped and its surviving prefix re-inserted (one GPU call)."""
        _need(0 <= n_leaves <= self.n_leaves, "rollback: target must not exceed the current leaf count")
        while self.n_leaves > n_leaves:
            have = self.n_leaves
            survivors = None
            # leaves of the newest batch start where the previous batch ended: read that from its undo record
            blob = self.store.get_raw(self._delta_key(self.n_batches))
            if blob is None:
                raise KeyError("Delta not found!")
            old_n = dict(self._unpack_delta(blob)).get(self.prefix + b"n")
            batch_start = int.from_bytes(old_n, "little") if old_n else 0
            if batch_start < n_leaves:
                survivors = [self.store.get_raw(self._key(0, i)) for i in range(batch_start, n_leaves)]
            self.pop_batch()
            assert self.n_leaves == batch_start < have
            if survivors:
                self.insert_batch(survivors)

    def root(self) -> bytes:
        return self._get(self.depth, 0)

    def path(self, idx: int):
        if not 0 <= idx < self.n_leaves:
            raise IndexError(f"leaf {idx} not in the tree ({self.n_leaves} leaves)")
        sibs, bits, i = [], 0, idx
        for lvl in range(self.depth):
            sibs.append(self._get(lvl, i ^ 1))
            bits |= (i & 1) << lvl
            i >>= 1
        return b"".join(sibs), bits

    def paths(self, indices):
        """Authentication paths of many leaves in the layout prove() takes: (siblings, path_bits) with siblings =
        len(indices) x depth x 32 bytes, proof-major, and one path_bits word per leaf."""
        got = [self.path(i) for i in indices]
        return b"".join(s for s, _ in got), [b for _, b in got]


def deposit_labeled(tree: MerkleTree, precommitments: bytes, tokens: bytes, amounts):
    """Append labeled deposits to the pool tree -> their labels.  The node assigns each deposit the next pool leaf index as
    its label, computes the leaf MultiMiMC7([precommitment, token, amount, label], 2) on the GPU from what the depositor sent
    (precommitments and tokens 32 bytes each, amounts uint64), and inserts the leaves in one insert_batch.  It never takes a
    leaf from the depositor: a label it did not assign cannot enter the pool."""
    _need(len(precommitments) % 32 == 0 and len(tokens) == len(precommitments),
          "deposit_labeled: precommitments and tokens must be equally long multiples of 32 bytes")
    n, start = len(precommitments) // 32, tree.n_leaves
    if start + n > (1 << tree.depth):
        raise OverflowError(f"tree of depth {tree.depth} holds {1 << tree.depth} leaves; {start} present, {n} more requested")
    labels = list(range(start, start + n))
    leaves = tree.ctx.labeled_leaves(precommitments, tokens, amounts, labels)
    tree.insert_batch([leaves[32 * k:32 * k + 32] for k in range(n)])
    return labels


def deposit_owned_labeled(tree: MerkleTree, precommitments: bytes, tokens: bytes, amounts):
    """Append owned labeled deposits to the pool tree -> their labels: deposit_labeled for owned labeled notes.  The node
    assigns each deposit the next pool leaf index as its label, computes the leaf MultiMiMC7([precommitment, token, amount,
    label], 7) on the GPU from what the depositor sent (precommitments MultiMiMC7([P, blinding], 6) and tokens 32 bytes each,
    amounts uint64), and inserts the leaves in one insert_batch.  It never takes a leaf from the depositor."""
    _need(len(precommitments) % 32 == 0 and len(tokens) == len(precommitments),
          "deposit_owned_labeled: precommitments and tokens must be equally long multiples of 32 bytes")
    n, start = len(precommitments) // 32, tree.n_leaves
    if start + n > (1 << tree.depth):
        raise OverflowError(f"tree of depth {tree.depth} holds {1 << tree.depth} leaves; {start} present, {n} more requested")
    labels = list(range(start, start + n))
    leaves = tree.ctx.owned_labeled_leaves(precommitments, tokens, amounts, labels)
    tree.insert_batch([leaves[32 * k:32 * k + 32] for k in range(n)])
    return labels


EXCLUSION_KEY_MAX = (1 << 32) + 1        # the blocklist tree's last key: above every note key (leaf index + 1 <= 2^32)


class ExclusionSet:
    """A compliance provider's blocklist of pool leaf indices as the exclusion statement's tree (DESIGN.md section 3).

    The flagged indices i_1 < ... < i_n (validated, sorted, deduplicated; each below 2^depth, at most 2^depth - 1 of them)
    give the keys k_0 = 0, k_j = i_j + 1, k_{n+1} = 2^32 + 1 and the leaves MultiMiMC7([k_j, k_{j+1}], 0), j = 0..n, in one
    og_mimc7_hash2 call; one MerkleTree.insert_batch of the pool's depth builds the tree on the GPU.  A new blocklist version
    is a new ExclusionSet.  witness(indices) gives what prove_exclusion takes for unflagged notes."""

    def __init__(self, ctx: Context, depth: int, flagged_indices, store=None):
        _need(1 <= depth <= 32, "ExclusionSet: depth must be in 1..32")
        flagged = sorted(set(int(i) for i in flagged_indices))
        _need(not flagged or (flagged[0] >= 0 and flagged[-1] < 1 << depth),
              f"ExclusionSet: flagged indices are pool leaf indices in [0, 2^{depth})")
        _need(len(flagged) < 1 << depth, f"ExclusionSet: a depth-{depth} tree holds at most 2^{depth} - 1 flagged indices")
        self.depth, self.flagged = depth, flagged
        self.keys = [0] + [i + 1 for i in flagged] + [EXCLUSION_KEY_MAX]
        self._flagged_set = frozenset(flagged)
        self.tree = MerkleTree(ctx, depth, store, prefix=b"xs/")
        _need(self.tree.n_leaves == 0, "ExclusionSet: the store already holds a blocklist tree")
        enc = lambda ks: b"".join(k.to_bytes(32, "little") for k in ks)
        leaves = ctx.mimc7_hash2(enc(self.keys[:-1]), enc(self.keys[1:]))
        self.tree.insert_batch([leaves[32 * j:32 * j + 32] for j in range(len(self.keys) - 1)])

    def root(self) -> bytes:
        return self.tree.root()

    def __contains__(self, index) -> bool:
        return index in self._flagged_set

    def __len__(self) -> int:
        return len(self.flagged)

    def witness(self, indices):
        """(excl_low, excl_next, excl_siblings, excl_path_bits) for the notes at pool leaf `indices`: the keys of the leaf
        that brackets each (lists of ints), its paths (len(indices) x depth x 32 bytes) and path words.  ValueError names
        any flagged index."""
        indices = [int(i) for i in indices]
        _need(all(0 <= i < 1 << self.depth for i in indices), f"ExclusionSet.witness: indices must be in [0, 2^{self.depth})")
        bad = sorted(set(i for i in indices if i in self._flagged_set))
        _need(not bad, f"ExclusionSet.witness: pool leaves {bad} are on the blocklist")
        js = [bisect.bisect_left(self.keys, i + 1) - 1 for i in indices]
        sibs, bits = self.tree.paths(js)
        return [self.keys[j] for j in js], [self.keys[j + 1] for j in js], sibs, bits


class ApprovedLabels:
    """A compliance provider's approved deposits as the labeled association statement's tree (DESIGN.md section 3).

    The approved labels (pool leaf indices, validated into [0, 2^depth), deduplicated and sorted) give the leaves label + 1,
    32 bytes little-endian, appended by one MerkleTree.insert_batch of the pool's depth, so the tree is hashed on the GPU;
    every other leaf is 0.  approve(labels) appends the labels not yet approved in one more insert_batch: a provider clears
    deposits as they arrive, and only the new leaves' ancestors are hashed.  witness(labels) gives what
    prove_labeled_association takes for approved labels."""

    def __init__(self, ctx: Context, depth: int, labels, store=None):
        _need(1 <= depth <= 32, "ApprovedLabels: depth must be in 1..32")
        self.depth = depth
        self.labels = []                                  # in leaf order
        self._leaf = {}                                   # label -> its leaf index
        self.tree = MerkleTree(ctx, depth, store, prefix=b"al/")
        _need(self.tree.n_leaves == 0, "ApprovedLabels: the store already holds an approved-label tree")
        self.approve(labels)

    def approve(self, labels):
        """Append the labels not yet approved (sorted) -> them."""
        labels = [int(x) for x in labels]
        _need(all(0 <= x < 1 << self.depth for x in labels), f"ApprovedLabels: labels are pool leaf indices in [0, 2^{self.depth})")
        new = sorted(set(x for x in labels if x not in self._leaf))
        self.tree.insert_batch([(x + 1).to_bytes(32, "little") for x in new])
        for x in new:
            self._leaf[x] = len(self.labels)
            self.labels.append(x)
        return new

    def root(self) -> bytes:
        return self.tree.root()

    def __contains__(self, label) -> bool:
        return label in self._leaf

    def __len__(self) -> int:
        return len(self.labels)

    def witness(self, labels):
        """(assoc_siblings, assoc_path_bits) for notes of `labels`: the paths of their leaves (len(labels) x depth x 32 bytes)
        and path words.  ValueError names every label that is not approved."""
        labels = [int(x) for x in labels]
        bad = sorted(set(x for x in labels if x not in self._leaf))
        _need(not bad, f"ApprovedLabels.witness: labels {bad} are not approved")
        return self.tree.paths([self._leaf[x] for x in labels])
