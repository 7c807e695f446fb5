"""The argument contract of the note entry points, one table over the seven note hashes and one over the twelve note
encryption and scan entry points, called through the C ABI: a batch of 0 is OG_OK, a null required pointer with a nonempty
batch is OG_E_INVALID, a scan takes at most 65 535 view keys, and the owned kinds' device scans refuse a non-canonical spend
public key with OG_E_ENCODING (their host scans are checked in test_owned_transfer.py and test_owned_labeled_transfer.py).
Every device pointer is a real allocation of the size the call would read, so no case depends on a check firing first."""
import ctypes as C

import pytest

from owshen_b200 import api
from oracle.bn254 import R

OG_E_ENCODING = -2
N = 3                              # items per nonempty batch

# og_<hash>(ctx, columns..., n, out): the bytes per item of each column in C ABI order
HASHES = {
    "labeled_precommitments": (32, 32),
    "labeled_leaves": (32, 32, 8, 4),
    "owned_public_keys": (32,),
    "owned_commitments": (32, 32, 32, 8),
    "owned_nullifiers": (32, 32, 4),
    "owned_labeled_precommitments": (32, 32),
    "owned_labeled_leaves": (32, 32, 8, 4),
}
# og_<kind>_encrypt(_dev)(ctx, inputs..., n, records, commitments, status): the bytes per note of each input
ENCRYPT_INPUTS = {
    "note": (32, 1, 32, 32, 32, 8, 32),
    "owned_note": (32, 1, 32, 32, 32, 8, 32),
    "owned_labeled_note": (32, 1, 32, 32, 32, 8, 4, 32),
}
ENCRYPT_OUTPUTS = (160, 32, 1)
SCAN_BUFFERS = (160, 32, 4, 128)   # records, commitments, owner, plaintexts
OWNED = {"note": False, "owned_note": True, "owned_labeled_note": True}


class Buffers:
    """Zeroed host (ctypes) or device (torch) buffers of the given byte sizes, as the pointers the entry points take."""

    def __init__(self, dev, sizes):
        if dev:
            import torch
            self._keep = [torch.zeros(max(s, 1), dtype=torch.uint8, device="cuda") for s in sizes]
            self.ptrs = [C.c_void_p(t.data_ptr()) for t in self._keep]
        else:
            self._keep = [C.create_string_buffer(max(s, 1)) for s in sizes]
            self.ptrs = [C.cast(b, C.c_void_p) for b in self._keep]


def with_null(ptrs, k):
    return ptrs[:k] + [None] + ptrs[k + 1:]


def hash_call(ctx, name, ptrs, n):
    """ptrs: the columns, then the output"""
    return getattr(api.lib(), f"og_{name}")(ctx._h, *ptrs[:-1], n, ptrs[-1])


def encrypt_call(ctx, kind, dev, ptrs, n):
    """ptrs: the inputs, then records, commitments, status"""
    fn = getattr(api.lib(), f"og_{kind}_encrypt" + ("_dev" if dev else ""))
    return fn(ctx._h, *ptrs[:-3], n, *ptrs[-3:])


def scan_call(ctx, kind, dev, keys, n_keys, ptrs, n):
    """keys: the host view keys (and spend public keys for the owned kinds); ptrs: records, commitments, owner, plaintexts"""
    fn = getattr(api.lib(), f"og_{kind}_scan" + ("_dev" if dev else ""))
    return fn(ctx._h, *keys, n_keys, ptrs[0], ptrs[1], n, ptrs[2], ptrs[3])


def scan_keys(kind, n_keys, view=5, spend=0):
    keys = [C.create_string_buffer(view.to_bytes(32, "little") * n_keys, max(32 * n_keys, 1))]
    if OWNED[kind]:
        keys.append(C.create_string_buffer(spend.to_bytes(32, "little") * n_keys, max(32 * n_keys, 1)))
    return keys


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HASHES))
def test_note_hash_arguments(ctx, name):
    sizes = [s * N for s in HASHES[name]] + [32 * N]
    ptrs = Buffers(False, sizes).ptrs
    assert hash_call(ctx, name, ptrs, 0) == api.OG_OK
    for k in range(len(ptrs)):
        assert hash_call(ctx, name, with_null(ptrs, k), N) == api.OG_E_INVALID, k


@pytest.mark.gpu
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind", sorted(ENCRYPT_INPUTS))
def test_note_encrypt_arguments(ctx, kind, dev):
    sizes = [s * N for s in ENCRYPT_INPUTS[kind] + ENCRYPT_OUTPUTS]
    ptrs = Buffers(dev, sizes).ptrs
    assert encrypt_call(ctx, kind, dev, ptrs, 0) == api.OG_OK
    for k in range(len(ptrs)):
        assert encrypt_call(ctx, kind, dev, with_null(ptrs, k), N) == api.OG_E_INVALID, k


@pytest.mark.gpu
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind", sorted(OWNED))
def test_note_scan_arguments(ctx, kind, dev):
    ptrs = Buffers(dev, [s * N for s in SCAN_BUFFERS]).ptrs
    keys = scan_keys(kind, 1)
    assert scan_call(ctx, kind, dev, keys, 1, ptrs, 0) == api.OG_OK
    assert scan_call(ctx, kind, dev, scan_keys(kind, 0), 0, ptrs, 0) == api.OG_OK
    for k in range(len(keys)):
        assert scan_call(ctx, kind, dev, with_null(keys, k), 1, ptrs, N) == api.OG_E_INVALID, ("key", k)
    for k in range(len(ptrs)):
        assert scan_call(ctx, kind, dev, keys, 1, with_null(ptrs, k), N) == api.OG_E_INVALID, k
    # the grid's y dimension holds the key index
    assert scan_call(ctx, kind, dev, scan_keys(kind, 65536), 65536, ptrs, N) == api.OG_E_INVALID
    if OWNED[kind] and dev:
        assert scan_call(ctx, kind, dev, scan_keys(kind, 1, spend=R), 1, ptrs, N) == OG_E_ENCODING
