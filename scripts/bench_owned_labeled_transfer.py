#!/usr/bin/env python
"""Owned labeled transfer proofs per second on one GPU, inputs resident in HBM (og_groth16_prove_owned_labeled_transfer_dev),
next to owned transfer proofs measured in the same run on the same card: the two statements share the note machinery, and the
owned labeled transfer has a third Merkle path and a domain twice as large at depth 32 (2^17 against 2^16).

Per statement: a depth-32 key from the development setup; per batch `--warmup` untimed steps, then `--steps` timed steps,
each one call for the whole batch, timed with CUDA events on the library stream; the median step gives proofs/s.  Then:
  - k_owned_labeled_transfer_witness and k_owned_transfer_witness over 1 024 proofs each in launches of their own (og_profile);
  - og_owned_labeled_note_scan_dev against og_owned_note_scan_dev over 2^20 records x 8 keys (median of --steps after
    --warmup), 1 in 1 000 records to one of the 8 wallets;
  - deposit_owned_labeled of 2^20 deposits into an empty depth-32 tree (median of --steps), host copies included.
The card's name, power limit and SM clock (nvidia-smi, read only) are printed with the results.
Usage: python scripts/bench_owned_labeled_transfer.py [--batch 1024 4096] [--steps 5] [--warmup 2] [--depth 32]"""
import argparse
import json
import os
import random
import statistics
import struct
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch

import owshen_b200 as ob
from owshen_b200 import api
from bench_g2_msm import gpu_info
from bench_owned_transfer import prove_rate as owned_prove_rate
from bench_transfer import device, device_fr, profile_step

R = ob.FR_MODULUS


def prove_rate(ctx, depth, batches, steps, warmup):
    """owned labeled transfer proofs/s at each batch: random inputs of the fifteen arrays (their proofs need not verify: the
    prover's work does not depend on it)."""
    rng = random.Random(7)
    PK = ob.ProvingKey(ctx, ob.setup_owned_labeled_transfer(ctx, depth, *[rng.randrange(1, R) for _ in range(5)])[0])
    fn = api.lib().og_groth16_prove_owned_labeled_transfer_dev
    out = []
    for batch in batches:
        rng = random.Random(batch)
        fr = lambda n: device_fr(rng, n)
        u64 = lambda n: device(struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)]))
        u32 = lambda n: device(struct.pack(f"<{n}I", *[rng.randrange(1 << depth) for _ in range(n)]))
        ins = [fr(batch), fr(batch), fr(batch), u64(batch), u32(batch), fr(2 * batch), fr(2 * batch), u64(2 * batch),
               fr(2 * depth * batch), u32(2 * batch), fr(2 * batch), fr(2 * batch), u64(2 * batch), fr(depth * batch), u32(batch)]
        rs = fr(2 * batch)
        proofs = torch.empty(256 * batch, dtype=torch.uint8, device="cuda")
        pub = torch.empty(288 * batch, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()

        def step():
            rc = fn(ctx._h, PK._h, *[t.data_ptr() for t in ins], batch, rs.data_ptr(), proofs.data_ptr(), pub.data_ptr())
            assert rc == 0, ob.OwshenB200Error(rc)

        for _ in range(warmup):
            step()
        ctx.sync()
        times = []
        for _ in range(steps):
            ctx.timer_start()
            step()
            times.append(ctx.timer_stop())
        out.append({"statement": "owned_labeled_transfer", "depth": depth, "batch": batch, "plan": PK.prover_plan(batch),
                    "ms_per_step": [round(t, 3) for t in times], "proofs_per_s": round(batch / (statistics.median(times) / 1e3), 1)})
        del ins, rs, proofs, pub
    PK.close()
    return out


def witness_kernels_ms(ctx, depth, batch):
    """k_owned_labeled_transfer_witness and k_owned_transfer_witness over `batch` proofs each in a launch of its own,
    alternated twice."""
    rng = random.Random(5)
    fr = lambda n: b"".join(rng.randrange(1 << 248).to_bytes(32, "little") for _ in range(n))
    u64 = lambda n: struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)])
    bits = lambda n: [rng.randrange(1 << depth) for _ in range(n)]
    o_in = (fr(batch), fr(batch), fr(batch), fr(2 * batch), fr(2 * batch), u64(2 * batch), fr(2 * depth * batch), bits(2 * batch),
            fr(2 * batch), fr(2 * batch), u64(2 * batch))
    l_in = o_in[:3] + (u64(batch), bits(batch)) + o_in[3:] + (fr(depth * batch), bits(batch))
    calls = (("k_owned_labeled_transfer_witness", lambda: ctx.owned_labeled_transfer_witness(depth, *l_in)),
             ("k_owned_transfer_witness", lambda: ctx.owned_transfer_witness(depth, *o_in)))
    out = {name: [] for name, _ in calls}
    for name, call in calls:
        call()
    for _ in range(2):
        for name, call in calls:
            out[name].append(profile_step(ctx, call).get(name))
    return out


def scan_ms(ctx, steps, warmup):
    """og_owned_labeled_note_scan_dev and og_owned_note_scan_dev over 2^20 records x 8 keys."""
    import numpy as np
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(2026)
    prng = random.Random(11)
    n = 1 << 20
    view = [prng.randrange(1, 1 << 248) for _ in range(8)]
    spend = [prng.randrange(1 << 248) for _ in range(8)]
    vb = b"".join(v.to_bytes(32, "little") for v in view)
    sp = ctx.owned_public_keys(b"".join(s.to_bytes(32, "little") for s in spend))
    foreign = b"".join(prng.randrange(1, 1 << 248).to_bytes(32, "little") for _ in range(64))
    px, odd = ctx.note_public_keys(vb + foreign)
    px = np.frombuffer(px, dtype=np.uint8).reshape(72, 32)
    odd = np.frombuffer(odd, dtype=np.uint8)
    dest = rng.integers(8, 72, size=n)
    dest[rng.choice(n, size=n // 1000, replace=False)] = rng.integers(0, 8, size=n // 1000)

    def rand_fr():
        a = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        a[:, 31] &= 31
        return a

    owners = rand_fr()
    mine = dest < 8
    owners[mine] = np.frombuffer(sp, dtype=np.uint8).reshape(8, 32)[dest[mine]]
    eph = rand_fr()
    eph[:, 0] |= 1
    to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).to(dev)
    d_in = [to_dev(px[dest]), to_dev(odd[dest]), to_dev(owners), to_dev(rand_fr()), to_dev(rand_fr()),
            to_dev(rng.integers(0, 1 << 63, size=n, dtype=np.uint64))]
    d_labels, d_eph = to_dev(rng.integers(0, 1 << 32, size=n, dtype=np.uint32)), to_dev(eph)
    recs = {k: (torch.empty(160 * n, dtype=torch.uint8, device=dev), torch.empty(32 * n, dtype=torch.uint8, device=dev))
            for k in ("labeled", "owned")}
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    ctx.owned_labeled_note_encrypt_dev(*d_in, d_labels, d_eph, n, *recs["labeled"], d_st)
    ctx.owned_note_encrypt_dev(*d_in, d_eph, n, *recs["owned"], d_st)
    d_owner = torch.empty(n, dtype=torch.int32, device=dev)
    d_plain = torch.empty(128 * n, dtype=torch.uint8, device=dev)
    ctx.sync()
    calls = {"og_owned_labeled_note_scan": lambda: ctx.owned_labeled_note_scan_dev(vb, sp, *recs["labeled"], n, d_owner, d_plain),
             "og_owned_note_scan": lambda: ctx.owned_note_scan_dev(vb, sp, *recs["owned"], n, d_owner, d_plain)}
    ms = {k: [] for k in calls}
    for _ in range(warmup):
        for call in calls.values():
            call()
    for _ in range(steps):                 # alternated, so both see the same clocks
        for k, call in calls.items():
            ctx.timer_start()
            call()
            ms[k].append(ctx.timer_stop())
    calls["og_owned_labeled_note_scan"]()
    ctx.sync()
    found = sum(1 for o in d_owner.cpu().tolist() if 0 <= o < 8)
    return {"records": n, "keys": 8, "owned_found": found, "expected_owned": int(mine.sum()),
            **{k: {"ms_median": round(statistics.median(v), 2), "ms": [round(x, 2) for x in v]} for k, v in ms.items()}}


def deposit_ms(ctx, steps, n=1 << 20):
    """deposit_owned_labeled of n deposits into an empty depth-32 tree: the key-7 leaves on the GPU and one insert_batch."""
    rng = random.Random(13)
    pre = b"".join(rng.randrange(1 << 248).to_bytes(32, "little") for _ in range(n))
    tokens = b"".join(rng.randrange(1 << 160).to_bytes(32, "little") for _ in range(n))
    amounts = struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)])
    times = []
    for _ in range(steps + 1):
        tree = ob.MerkleTree(ctx, 32)
        ctx.sync()
        t0 = time.perf_counter()
        labels = ob.deposit_owned_labeled(tree, pre, tokens, amounts)
        tree.root()
        ctx.sync()
        times.append((time.perf_counter() - t0) * 1e3)
        assert labels[-1] == n - 1
        del tree
    return {"deposits": n, "ms_median": round(statistics.median(times[1:]), 1), "ms": [round(t, 1) for t in times[1:]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--depth", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_owned_labeled_transfer: no CUDA device")
    info = gpu_info()
    for stmt in ("owned_labeled_transfer", "owned_transfer", "owned_labeled_transfer", "owned_transfer"):
        ctx = ob.Context(0)                # a context per pass: one prover's scratch lanes are released before the next's
        rows = (prove_rate(ctx, args.depth, args.batch, args.steps, args.warmup) if stmt == "owned_labeled_transfer"
                else owned_prove_rate(ctx, stmt, args.depth, args.batch, args.steps, args.warmup))
        for r in rows:
            print(json.dumps(dict(r, gpu=info)), flush=True)
        ctx.close()
    ctx = ob.Context(0)
    print(json.dumps({"witness_kernels_ms": witness_kernels_ms(ctx, args.depth, min(args.batch)), "batch": min(args.batch),
                      "depth": args.depth, "gpu": info}), flush=True)
    print(json.dumps({"scan": scan_ms(ctx, args.steps, args.warmup), "gpu": gpu_info()}), flush=True)
    print(json.dumps({"deposit_owned_labeled": deposit_ms(ctx, args.steps), "gpu": gpu_info()}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
