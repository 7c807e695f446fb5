"""ctypes binding of libowshen_b200.so and the host-side mirror of the API BASELINE.json's north_star
names: prove() / verify() / MerkleTree.  The reference (OwshenNetwork/owshen @ c7b1f00) has no such
API (SURVEY.md section 0), so names and error behaviour follow its conventions instead: fallible
calls raise (anyhow::Result -> exception), byte blobs are owned `bytes`, field elements are 32-byte
little-endian (/root/reference/src/blockchain/tx/owshen_airdrop/babyjubjub/mod.rs:7-11).

All hashing, witness generation, NTTs and MSMs run in the CUDA library; nothing here computes.
"""
import array
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


def _transfer_args(fn, batch, depth, roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings, in_path_bits,
                   out_nullifiers, out_secrets, out_amounts):
    """Length checks of a transfer batch's eleven input arrays -> their pointers in C ABI order."""
    amounts = [_u64_array(in_amounts), _u64_array(out_amounts)]
    bits = _u32_array(in_path_bits)
    for name, buf, size in (("roots", roots, 32), ("tokens", tokens, 32), ("recipients", recipients, 32),
                            ("in_nullifiers", in_nullifiers, 64), ("in_secrets", in_secrets, 64), ("in_amounts", amounts[0], 16),
                            ("in_siblings", in_siblings, 64 * depth), ("in_path_bits", bits, 8),
                            ("out_nullifiers", out_nullifiers, 64), ("out_secrets", out_secrets, 64), ("out_amounts", amounts[1], 16)):
        if isinstance(buf, C.Array):        # converted from a sequence above
            _need(C.sizeof(buf) == size * batch, f"{fn}: {name}: expected {size * batch // C.sizeof(buf._type_)} values, got {len(buf)}")
        else:
            _need_len(buf, size * batch, f"{fn}: {name}")
    return [_ptr(x) for x in (roots, tokens, recipients, in_nullifiers, in_secrets, amounts[0], in_siblings, bits,
                              out_nullifiers, out_secrets, amounts[1])]


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
    FIELD_PROBE_OPS = {"g1": ("mul", "sqr", "sub", "dbl"),
                       "g2": ("mul_lazy", "sqr_lazy", "add_lazy", "sub_lazy", "canonical", "mul", "sqr", "is_zero_lazy")}

    def field_probe_raw(self, unit: str, op: str, a: bytes, b: bytes = None) -> bytes:
        """Test/debug probe: element-wise arithmetic of the G1 ("g1": Fq, 32 B per operand) or G2 ("g2": Fq2, 64 B) MSM unit on
        raw Montgomery limbs, through the functions its bucket kernels call (the probe kernel's own compiled copies); raw limbs out."""
        _need(unit in self.FIELD_PROBE_OPS and op in self.FIELD_PROBE_OPS[unit], "field_probe_raw: unknown unit or op")
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
        n = len(pk_is_odd)
        if ephemerals is None:
            ephemerals = b"".join(fr_bytes(_rand.randbelow(NOTE_SUBGROUP_ORDER - 1) + 1) for _ in range(n))
        am = _u64_array(amounts)
        for name, buf in (("pk_x", pk_x), ("nullifiers", nullifiers), ("secrets", secrets), ("tokens", tokens), ("ephemerals", ephemerals)):
            _need(len(buf) == 32 * n, f"note_encrypt: {name}: expected {32 * n} bytes, got {len(buf)}")
        _need((C.sizeof(am) if isinstance(am, C.Array) else _blen(am)) == 8 * n, "note_encrypt: expected one amount per note")
        rec, cm, st = C.create_string_buffer(160 * n), C.create_string_buffer(32 * n), C.create_string_buffer(n)
        _check(lib().og_note_encrypt(self._h, pk_x, pk_is_odd, nullifiers, secrets, tokens, _ptr(am), ephemerals, n, rec, cm, st), self)
        return rec.raw, cm.raw, st.raw[:n]

    def note_encrypt_dev(self, d_pk_x, d_pk_is_odd, d_nullifiers, d_secrets, d_tokens, d_amounts, d_ephemerals, n: int,
                         d_out_records, d_out_commitments, d_out_status):
        """og_note_encrypt_dev: device buffers (addresses or tensors), enqueued on the context's stream."""
        _check(lib().og_note_encrypt_dev(self._h, *[_ptr(x) for x in (d_pk_x, d_pk_is_odd, d_nullifiers, d_secrets, d_tokens, d_amounts,
                                                                     d_ephemerals)], n,
                                         *[_ptr(x) for x in (d_out_records, d_out_commitments, d_out_status)]), self)

    def note_scan(self, view_keys: bytes, records: bytes, commitments: bytes):
        """Trial-decrypt every record under every view key -> (owners, plaintexts): owners[i] is the lowest index of a key
        that owns record i, NOTE_NOT_OWNED or NOTE_MALFORMED; plaintexts holds 128 bytes per record (nullifier, secret, token,
        amount), zero unless owned."""
        _need(len(view_keys) % 32 == 0, "note_scan: view keys must be a multiple of 32 bytes")
        _need(len(records) % 160 == 0, "note_scan: records must be a multiple of 160 bytes")
        n = len(records) // 160
        _need(len(commitments) == 32 * n, "note_scan: expected one 32-byte commitment per record")
        owner, plain = (C.c_uint32 * n)(), C.create_string_buffer(128 * n)
        _check(lib().og_note_scan(self._h, view_keys, len(view_keys) // 32, records, commitments, n, owner, plain), self)
        return list(owner), plain.raw

    def note_scan_dev(self, view_keys: bytes, d_records, d_commitments, n: int, d_out_owner, d_out_plaintexts):
        """og_note_scan_dev: view keys on the host, every other buffer on the device, enqueued on the context's stream."""
        _need(len(view_keys) % 32 == 0, "note_scan_dev: view keys must be a multiple of 32 bytes")
        _check(lib().og_note_scan_dev(self._h, view_keys, len(view_keys) // 32, _ptr(d_records), _ptr(d_commitments), n,
                                      _ptr(d_out_owner), _ptr(d_out_plaintexts)), self)

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

    def withdraw_witness(self, depth, nullifiers: bytes, secrets: bytes, recipients: bytes, siblings: bytes, path_bits) -> bytes:
        _need(len(nullifiers) % 32 == 0 and 1 <= depth <= 32, "withdraw_witness: bad nullifiers length or depth")
        n = len(nullifiers) // 32
        _need(len(secrets) == 32 * n and len(recipients) == 32 * n and len(siblings) == 32 * n * depth and len(path_bits) == n,
              "withdraw_witness: secrets / recipients / siblings / path_bits do not match the batch")
        nv = r1cs_info(depth)["n_vars"]
        out = C.create_string_buffer(32 * n * nv)
        _check(lib().og_withdraw_witness(self._h, depth, nullifiers, secrets, recipients, siblings, _bits_array(path_bits), n, out), self)
        return out.raw

    def deposit_witness(self, nullifiers: bytes, secrets: bytes, depositors: bytes) -> bytes:
        """Full assignments of the deposit statement, n_vars * 32 bytes per deposit, computed on the GPU."""
        _need(len(nullifiers) % 32 == 0, "deposit_witness: nullifiers must be a multiple of 32 bytes")
        n = len(nullifiers) // 32
        _need(len(secrets) == 32 * n and len(depositors) == 32 * n, "deposit_witness: secrets / depositors do not match the batch")
        nv = deposit_r1cs_info()["n_vars"]
        out = C.create_string_buffer(32 * n * nv)
        _check(lib().og_deposit_witness(self._h, nullifiers, secrets, depositors, n, out), self)
        return out.raw

    def transfer_witness(self, depth, roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings, in_path_bits,
                         out_nullifiers, out_secrets, out_amounts) -> bytes:
        """Full assignments of the depth-`depth` transfer statement, n_vars * 32 bytes per transfer, computed on the GPU.
        Per transfer: roots / tokens / recipients 32 bytes each; in_* / out_* note 0 then note 1 (nullifiers and secrets
        2 x 32 bytes, amounts 2 x uint64 as 8-byte little-endian buffers, uint64 arrays or ints); in_siblings 2 * depth
        elements (input 0's path, then input 1's); in_path_bits 2 words."""
        _need(1 <= depth <= 32 and _blen(roots) is not None and _blen(roots) % 32 == 0,
              "transfer_witness: depth must be 1..32 and roots a multiple of 32 bytes")
        n = _blen(roots) // 32
        args = _transfer_args("transfer_witness", n, depth, roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts,
                              in_siblings, in_path_bits, out_nullifiers, out_secrets, out_amounts)
        nv = transfer_r1cs_info(depth)["n_vars"]
        out = C.create_string_buffer(32 * n * nv)
        _check(lib().og_transfer_witness(self._h, depth, *args, n, out), self)
        return out.raw


def mimc7_constants():
    out = C.create_string_buffer(32 * 91)
    n = C.c_uint32()
    _check(lib().og_mimc7_constants(out, C.byref(n)))
    return [int.from_bytes(out.raw[32 * i:32 * i + 32], "little") for i in range(n.value)]


def r1cs_info(depth: int) -> dict:
    v = [C.c_uint32() for _ in range(4)]
    _check(lib().og_withdraw_r1cs_info(depth, *[C.byref(x) for x in v]))
    return dict(n_constraints=v[0].value, n_vars=v[1].value, n_pub=v[2].value, log_m=v[3].value)


def r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's withdraw R1CS."""
    w = "ABC".index(which)
    nnz = C.c_uint64()
    _check(lib().og_withdraw_r1cs_export(depth, w, None, None, None, C.byref(nnz)))
    nc = r1cs_info(depth)["n_constraints"]
    ptr = (C.c_uint32 * (nc + 1))()
    col = (C.c_uint32 * nnz.value)()
    val = C.create_string_buffer(32 * nnz.value)
    _check(lib().og_withdraw_r1cs_export(depth, w, ptr, col, val, C.byref(nnz)))
    return list(ptr), list(col), [int.from_bytes(val.raw[32 * i:32 * i + 32], "little") for i in range(nnz.value)]


def deposit_r1cs_info() -> dict:
    v = [C.c_uint32() for _ in range(4)]
    _check(lib().og_deposit_r1cs_info(*[C.byref(x) for x in v]))
    return dict(n_constraints=v[0].value, n_vars=v[1].value, n_pub=v[2].value, log_m=v[3].value)


def deposit_r1cs_export(which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's deposit R1CS."""
    w = "ABC".index(which)
    nnz = C.c_uint64()
    _check(lib().og_deposit_r1cs_export(w, None, None, None, C.byref(nnz)))
    nc = deposit_r1cs_info()["n_constraints"]
    ptr = (C.c_uint32 * (nc + 1))()
    col = (C.c_uint32 * nnz.value)()
    val = C.create_string_buffer(32 * nnz.value)
    _check(lib().og_deposit_r1cs_export(w, ptr, col, val, C.byref(nnz)))
    return list(ptr), list(col), [int.from_bytes(val.raw[32 * i:32 * i + 32], "little") for i in range(nnz.value)]


def transfer_r1cs_info(depth: int) -> dict:
    v = [C.c_uint32() for _ in range(4)]
    _check(lib().og_transfer_r1cs_info(depth, *[C.byref(x) for x in v]))
    return dict(n_constraints=v[0].value, n_vars=v[1].value, n_pub=v[2].value, log_m=v[3].value)


def transfer_r1cs_export(depth: int, which: str):
    """(row_ptr, col_idx, coeffs as ints) of matrix 'A' | 'B' | 'C' of the product's depth-`depth` transfer R1CS."""
    w = "ABC".index(which)
    nnz = C.c_uint64()
    _check(lib().og_transfer_r1cs_export(depth, w, None, None, None, C.byref(nnz)))
    nc = transfer_r1cs_info(depth)["n_constraints"]
    ptr = (C.c_uint32 * (nc + 1))()
    col = (C.c_uint32 * nnz.value)()
    val = C.create_string_buffer(32 * nnz.value)
    _check(lib().og_transfer_r1cs_export(depth, w, ptr, col, val, C.byref(nnz)))
    return list(ptr), list(col), [int.from_bytes(val.raw[32 * i:32 * i + 32], "little") for i in range(nnz.value)]


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


def setup_deposit(ctx: Context, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the deposit statement -> (pk_bytes, vk_bytes): its exported R1CS through setup_r1cs."""
    info = deposit_r1cs_info()
    return setup_r1cs(ctx, info["n_vars"], info["n_pub"], *(deposit_r1cs_export(m) for m in "ABC"), tau, alpha, beta, gamma, delta)


def setup_transfer(ctx: Context, depth: int, tau: int, alpha: int, beta: int, gamma: int, delta: int):
    """Development setup of the depth-`depth` transfer statement -> (pk_bytes, vk_bytes): its exported R1CS through
    setup_r1cs.  The key records depth 0; the prover recognises it as a transfer key by its shape."""
    info = transfer_r1cs_info(depth)
    return setup_r1cs(ctx, info["n_vars"], info["n_pub"], *(transfer_r1cs_export(depth, m) for m in "ABC"),
                      tau, alpha, beta, gamma, delta)


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


def ptau_prepare_deposit(ctx: Context, acc: bytes):
    info = deposit_r1cs_info()
    return ptau_prepare(ctx, acc, info["n_vars"], info["n_pub"], *(deposit_r1cs_export(m) for m in "ABC"))


def ptau_prepare_transfer(ctx: Context, acc: bytes, depth: int):
    info = transfer_r1cs_info(depth)
    return ptau_prepare(ctx, acc, info["n_vars"], info["n_pub"], *(transfer_r1cs_export(depth, m) for m in "ABC"))


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

    def prove_withdraw(self, nullifiers, secrets, recipients, siblings, path_bits, rs, want_public=True):
        """Host buffers in, host buffers out (H2D / D2H inside).  Buffers may be bytes or pinned
        tensors / arrays exposing data_ptr() / .ctypes.  Returns (proofs, public_inputs)."""
        batch = len(path_bits)
        _need(self.depth >= 1, "prove_withdraw: this key was not made for the withdraw statement")
        for name, buf, size in (("nullifiers", nullifiers, 32), ("secrets", secrets, 32), ("recipients", recipients, 32),
                                ("siblings", siblings, 32 * self.depth), ("rs", rs, 64)):
            _need_len(buf, size * batch, f"prove_withdraw: {name}")
        bits = path_bits if hasattr(path_bits, "data_ptr") or hasattr(path_bits, "ctypes") else _bits_array(path_bits)
        proofs = C.create_string_buffer(PROOF_BYTES * batch)
        pub = C.create_string_buffer(32 * self.n_pub * batch) if want_public else None
        _check(lib().og_groth16_prove_withdraw(self.ctx._h, self._h, _ptr(nullifiers), _ptr(secrets), _ptr(recipients),
                                               _ptr(siblings), _ptr(bits), batch, _ptr(rs), proofs, pub), self.ctx)
        return proofs.raw, (pub.raw if want_public else None)

    def prove_deposit(self, nullifiers, secrets, depositors, rs, want_public=True):
        """Batch of deposit proofs from the secret inputs (witness generation on the GPU).  Buffers as in prove_withdraw;
        returns (proofs, public_inputs) with public inputs (commitment, depositor) per proof."""
        _need(_blen(rs) is not None and _blen(rs) % 64 == 0, "prove_deposit: rs must be a buffer of 64 bytes (r, s) per proof")
        batch = _blen(rs) // 64
        for name, buf in (("nullifiers", nullifiers), ("secrets", secrets), ("depositors", depositors)):
            _need_len(buf, 32 * batch, f"prove_deposit: {name}")
        proofs = C.create_string_buffer(PROOF_BYTES * batch)
        pub = C.create_string_buffer(32 * self.n_pub * batch) if want_public else None
        _check(lib().og_groth16_prove_deposit(self.ctx._h, self._h, _ptr(nullifiers), _ptr(secrets), _ptr(depositors), batch,
                                              _ptr(rs), proofs, pub), self.ctx)
        return proofs.raw, (pub.raw if want_public else None)

    @property
    def transfer_depth(self):
        """The depth d whose transfer statement has this key's shape (transfer_r1cs_info), or None."""
        for d in range(1, 33):
            info = transfer_r1cs_info(d)
            if (info["n_vars"], info["n_pub"]) == (self.n_vars, self.n_pub):
                return d
        return None

    def prove_transfer(self, roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts, in_siblings, in_path_bits,
                       out_nullifiers, out_secrets, out_amounts, rs, want_public=True):
        """Batch of transfer proofs from the notes (witness generation on the GPU).  Inputs as in Context.transfer_witness;
        returns (proofs, public_inputs) with public inputs (root, public_amount, token, recipient, nullifier_hash[2],
        out_commitment[2]) per proof."""
        depth = self.transfer_depth
        if depth is None:
            raise OwshenB200Error(OG_E_INVALID, "prove_transfer: this key was not made for a transfer statement")
        _need(_blen(rs) is not None and _blen(rs) % 64 == 0, "prove_transfer: rs must be a buffer of 64 bytes (r, s) per proof")
        batch = _blen(rs) // 64
        args = _transfer_args("prove_transfer", batch, depth, roots, tokens, recipients, in_nullifiers, in_secrets, in_amounts,
                              in_siblings, in_path_bits, out_nullifiers, out_secrets, out_amounts)
        proofs = C.create_string_buffer(PROOF_BYTES * batch)
        pub = C.create_string_buffer(32 * self.n_pub * batch) if want_public else None
        _check(lib().og_groth16_prove_transfer(self.ctx._h, self._h, *args, batch, _ptr(rs), proofs, pub), self.ctx)
        return proofs.raw, (pub.raw if want_public else None)

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
