"""C-ABI checks that need no GPU: the library loads, exports every symbol include/owshen_b200.h declares,
refuses to run without a device (no CPU fallback), and its host-side logic (withdraw R1CS builder, MiMC7
constant derivation, Groth16 verifier) agrees with the oracle."""
import os
import random
import re

import pytest

import owshen_b200 as ob
from owshen_b200 import api
from oracle import bn254 as bn
from oracle import cport, mimc7
from oracle.withdraw_circuit import build_r1cs, witness
from tests.helpers import vk_blob

R = bn.R
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_declared_symbol_is_exported():
    hdr = open(os.path.join(ROOT, "include", "owshen_b200.h")).read()
    declared = set(re.findall(r"\b(og_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "header parse failed"
    L = ob.lib()
    for name in sorted(declared):
        assert hasattr(L, name), f"{name} declared in include/owshen_b200.h but not exported"
    assert declared == set(api.ABI_SYMBOLS), declared ^ set(api.ABI_SYMBOLS)
    assert L.og_abi_version() == 1


def test_library_is_built_for_sm90a_only():
    """The kernels are compiled for the H100 (sm_90a) and nothing else: code for another architecture does not load
    there, and a stale build for one would fail only at the first kernel launch."""
    import shutil
    import subprocess
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "--list-elf", api._LIB_PATH], capture_output=True, text=True, check=True).stdout
    archs = set(re.findall(r"\.(sm_\w+)\.cubin", out))
    assert archs == {"sm_90a"}, out


def test_header_prototypes_match_the_ctypes_mirror():
    """Parameter counts (and pointer-ness of every parameter) of include/owshen_b200.h against api.ABI_SYMBOLS:
    a drifted mirror would pass garbage across the boundary without any loader error."""
    import ctypes as C
    hdr = open(os.path.join(ROOT, "include", "owshen_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    protos = dict(re.findall(r"\b(og_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr))
    assert set(protos) == set(api.ABI_SYMBOLS)
    for name, params in protos.items():
        params = params.strip()
        plist = [] if params in ("", "void") else [x.strip() for x in params.split(",")]
        res, args = api._SIGS[name]
        assert len(plist) == len(args), f"{name}: header has {len(plist)} parameters, api.py {len(args)}"
        for decl, ct in zip(plist, args):
            is_ptr_c = "*" in decl
            is_ptr_py = ct in (C.c_void_p, C.c_char_p) or isinstance(ct, type) and issubclass(ct, C._Pointer)
            assert is_ptr_c == is_ptr_py, f"{name}: `{decl}` vs {ct}"
            if not is_ptr_c:
                width = 8 if "64" in decl else 4
                assert C.sizeof(ct) == width, f"{name}: `{decl}` vs {ct}"


def test_rust_bindings_are_in_step_with_the_header():
    """bindings/rust/ffi.rs is generated from include/owshen_b200.h (scripts/gen_rust_ffi.py); it cannot be compiled
    here (no rustc), so at least it must not drift."""
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gen_rust_ffi.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    ffi = open(os.path.join(ROOT, "bindings", "rust", "ffi.rs")).read()
    assert ffi.count("pub fn og_") == len(api.ABI_SYMBOLS)
    wrapper = open(os.path.join(ROOT, "bindings", "rust", "prover.rs")).read()
    for used in set(re.findall(r"ffi::(og_[a-z0-9_]+)", wrapper)):
        assert f"pub fn {used}(" in ffi, used


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(ob.OwshenB200Error) as e:
        ob.Context(0)
    assert e.value.code == -3


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "owshen_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f
                assert '#include "../../oracle' not in src and "liboracle" not in src, f


def test_mimc_constants_derived_by_the_product():
    assert api.mimc7_constants() == mimc7.CONSTANTS


@pytest.mark.parametrize("depth", [1, 2, 32])
def test_withdraw_r1cs_matches_spec(depth):
    cs = build_r1cs(depth)
    info = api.r1cs_info(depth)
    assert (info["n_constraints"], info["n_vars"], info["n_pub"]) == (cs.n_constraints, cs.n_vars, cs.n_pub)
    for m in "ABC":
        ptr, col, val = api.r1cs_export(depth, m)
        eptr, ecol, eval_ = cs.csr(m)
        assert ptr == eptr and col == ecol and val == eval_, m


def test_host_verifier_accepts_oracle_proof_and_rejects_tampering():
    rng = random.Random(9)
    depth = 4
    cs = build_r1cs(depth)
    pkb, vkb = cport.setup_bytes(cs, *[rng.randrange(1, R) for _ in range(5)])
    sib = [rng.randrange(R) for _ in range(depth)]
    w = witness(11, 22, 33, sib, [1, 0, 1, 1])
    pr = cport.Prover(cs, pkb)
    proof = pr.prove(cport.frs(w), 5, 7)
    vk = vk_blob(vkb)
    pub = cport.frs(w[1:4])
    assert ob.verify(vk, pub, proof)
    bad = bytearray(pub); bad[0] ^= 1
    assert not ob.verify(vk, bytes(bad), proof)
    other = pr.prove(cport.frs(w), 6, 7)
    assert ob.verify(vk, pub, other)
    assert not ob.verify(vk, pub, proof[:64] + other[64:])
    with pytest.raises(ob.OwshenB200Error):
        ob.verify(vk, pub, b"\xff" * 256)          # non-canonical coordinates
    with pytest.raises(ob.OwshenB200Error):
        ob.verify(vk[:-1], pub, proof)
    # a point that is on the curve but the proof is garbage -> False, not an exception
    g1, g2 = bn.g1_to_bytes(bn.G1_GEN), bn.g2_to_bytes(bn.G2_GEN)
    assert not ob.verify(vk, pub, g1 + g2 + g1)


def test_kvstore_shape_matches_reference_trait():
    # /root/reference/src/db/mod.rs:24-52: get_raw, batch_put_raw, None deletes
    s = ob.RamKvStore()
    s.batch_put_raw([(b"k1", b"v1"), (b"k2", b"v2")])
    assert s.get_raw(b"k1") == b"v1" and s.get_raw(b"missing") is None
    s.batch_put_raw([(b"k1", None)])
    assert s.get_raw(b"k1") is None and s.get_raw(b"k2") == b"v2"


def test_external_encodings_round_trip():
    """EIP-197 calldata layout and snarkjs JSON of the library's proof / vk blobs (pure byte shuffling)."""
    import json
    from owshen_b200 import formats
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "vectors.json")))["groth16"]
    proof = bytes.fromhex(g["proof"])
    ev = formats.proof_to_eip197(proof)
    assert len(ev) == 256 and formats.proof_from_eip197(ev) == proof
    (ax, ay), ((bx0, bx1), (by0, by1)), (cx, cy) = formats.proof_points(proof)
    assert int.from_bytes(ev[:32], "big") == ax and int.from_bytes(ev[64:96], "big") == bx1 and int.from_bytes(ev[96:128], "big") == bx0
    assert bn.g1_on_curve((ax, ay)) and bn.g1_on_curve((cx, cy)) and bn.g2_on_curve(((bx0, bx1), (by0, by1)))
    sj = formats.proof_to_snarkjs(proof)
    assert sj["pi_a"] == [str(ax), str(ay), "1"] and sj["pi_b"][0] == [str(bx0), str(bx1)]
    v = g["vk"]
    vk = b"OGVK" + (1).to_bytes(4, "little") + (3).to_bytes(4, "little") + bytes.fromhex(v["alpha1"] + v["beta2"] + v["gamma2"] + v["delta2"] + v["ic"])
    p = formats.parse_vk(vk)
    assert p["n_pub"] == 3 and len(p["ic"]) == 4 and all(bn.g1_on_curve(q) for q in p["ic"]) and bn.g2_on_curve(p["delta2"])
    assert formats.vk_to_snarkjs(vk)["nPublic"] == 3
    pub = b"".join(bn.fr_to_bytes(int(x)) for x in g["public"])
    assert formats.public_inputs_to_eip197(pub)[:32] == int(g["public"][0]).to_bytes(32, "big")
    assert ob.verify(vk, pub, proof)
