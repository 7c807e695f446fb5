"""The batched prover's digit sort (msm.cu: k_sort_part_count, k_sort_part_scatter, k_sort_local) on digit distributions
that pile up in one partition and one bucket, compared byte for byte with the oracle's C prover.

The sort splits each proof's digits into coarse partitions (the top bits of the bucket id) and sorts every partition in
shared memory.  Private witness values in {0, 1, 2} give every window but the first a zero digit and put nearly every digit
of the A and B MSMs in buckets 0 and 1, i.e. in one partition of one proof; an all-zero witness with r = s = 0 leaves every
partition empty.  Proofs are deterministic in (pk, witness, r, s), so the same witnesses proved in other chunkings must give
the same bytes."""
import random

import pytest

import owshen_b200 as ob
from oracle import bn254 as bn
from oracle import cport
from tests.helpers import rand_inputs, withdraw_keys32

R = bn.R
SORT_KERNELS = ("k_sort_part_count", "k_sort_part_scatter", "k_sort_local")


@pytest.fixture(scope="module")
def keys32(ctx):
    return withdraw_keys32(ctx)


def small_witness(rng, cs, values=(0, 1, 2)):
    """w_0 = 1, public inputs random, every private value drawn from `values`."""
    w = [1] + [rng.randrange(R) for _ in range(cs.n_pub)] + [rng.choice(values) for _ in range(cs.n_vars - cs.n_pub - 1)]
    return cport.frs(w)


def random_witness(rng, cs):
    nul, sec, rec, sib, bits = rand_inputs(rng, 1, 32)
    return cport.withdraw_witness(nul, sec, rec, sib, bits, 32)


def prove(ctx, pk, wit, rs, monkeypatch, chunk=None, lanes=None):
    for k, v in (("OG_CHUNK", chunk), ("OG_LANES", lanes)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))
    PK = ob.ProvingKey(ctx, pk)
    try:
        ctx.profile(True)
        proofs = PK.prove_witnesses(wit, rs)
        ctx.sync()
        ctx.profile(False)
        prof = ctx.profile_dump()
    finally:
        PK.close()
    return proofs, prof


def check_against_oracle(cs, pkb, wits, rs, proofs, idx):
    n = 32 * cs.n_vars
    exp = cport.Prover(cs, pkb).prove_batch(b"".join(wits[i] for i in idx), b"".join(rs[64 * i:64 * i + 64] for i in idx))
    for k, i in enumerate(idx):
        assert proofs[256 * i:256 * i + 256] == exp[256 * k:256 * k + 256], i
    assert all(len(w) == n for w in wits)


@pytest.mark.gpu
def test_prover_sort_small_witness_values(ctx, keys32, monkeypatch):
    """Every proof of the batch has private values in {0, 1, 2}: almost every digit of A and B lands in one partition."""
    pk, vk, cs, pkb, vkb = keys32
    rng = random.Random(71)
    wits = [small_witness(rng, cs) for _ in range(4)]
    rs = cport.frs([rng.randrange(R) for _ in range(8)])
    proofs, prof = prove(ctx, pk, b"".join(wits), rs, monkeypatch)
    # three MSMs per chunk, each through the partitioned sort and none through the one-shot scatter
    assert all(prof.get(k, (0, 0))[0] == 3 for k in SORT_KERNELS), prof
    assert "k_digits_scatter" not in prof and "k_digits_count" not in prof
    check_against_oracle(cs, pkb, wits, rs, proofs, [0, 3])


@pytest.mark.gpu
def test_prover_sort_all_zero_witness(ctx, keys32, monkeypatch):
    """An all-zero witness with r = s = 0: the only non-zero scalars are the fixed terms, every other partition is empty."""
    pk, vk, cs, pkb, vkb = keys32
    wits = [bytes(32 * cs.n_vars)] * 2
    rs = bytes(128)
    proofs, _ = prove(ctx, pk, b"".join(wits), rs, monkeypatch)
    assert proofs[:256] == proofs[256:]
    check_against_oracle(cs, pkb, wits, rs, proofs, [0])


@pytest.mark.gpu
def test_prover_sort_mixed_batch(ctx, keys32, monkeypatch):
    """Skewed, empty and random witnesses in one batch; the same bytes in one chunk, and in chunks of 3 on two lanes."""
    pk, vk, cs, pkb, vkb = keys32
    rng = random.Random(72)
    kinds = ["small", "random", "zero", "bits", "random", "small", "random", "bits"]
    wits = []
    for k in kinds:
        if k == "small":
            wits.append(small_witness(rng, cs))
        elif k == "bits":
            wits.append(small_witness(rng, cs, (0, 1)))
        elif k == "zero":
            wits.append(bytes(32 * cs.n_vars))
        else:
            wits.append(random_witness(rng, cs))
    rs = bytearray(cport.frs([rng.randrange(R) for _ in range(2 * len(kinds))]))
    rs[128:192] = bytes(64)                                  # the zero witness gets r = s = 0
    rs = bytes(rs)
    proofs, _ = prove(ctx, pk, b"".join(wits), rs, monkeypatch)
    check_against_oracle(cs, pkb, wits, rs, proofs, [0, 1, 2, 3])
    again, _ = prove(ctx, pk, b"".join(wits), rs, monkeypatch, chunk=3, lanes=2)
    assert again == proofs
