#!/usr/bin/env python
"""Ragequit proofs per second on one GPU, inputs resident in HBM (og_groth16_prove_ragequit_dev), next to owned labeled
transfer proofs measured in the same run on the same card: a ragequit spends one owned labeled note with one Merkle path,
and its domain at depth 32 is 2^15 against the owned labeled transfer's 2^17.

Per statement: a depth-32 key from the development setup; per batch `--warmup` untimed steps, then `--steps` timed steps,
each one call for the whole batch, timed with CUDA events on the library stream; the median step gives proofs/s.  The two
statements are alternated twice.  Then k_ragequit_witness and k_owned_labeled_transfer_witness over the smallest batch
(1 024 proofs by default) each in launches of their own (og_profile), alternated twice.
The card's name, power limit and SM clock (nvidia-smi, read only) are printed with the results.
Usage: python scripts/bench_ragequit.py [--batch 1024 4096] [--steps 5] [--warmup 2] [--depth 32]"""
import argparse
import json
import os
import random
import statistics
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch

import owshen_b200 as ob
from owshen_b200 import api
from bench_g2_msm import gpu_info
from bench_owned_labeled_transfer import prove_rate as olt_prove_rate
from bench_transfer import device, device_fr, profile_step

R = ob.FR_MODULUS


def prove_rate(ctx, depth, batches, steps, warmup):
    """ragequit proofs/s at each batch: random inputs of the nine arrays (their proofs need not verify: the prover's work does
    not depend on it)."""
    rng = random.Random(7)
    PK = ob.ProvingKey(ctx, ob.setup_ragequit(ctx, depth, *[rng.randrange(1, R) for _ in range(5)])[0])
    fn = api.lib().og_groth16_prove_ragequit_dev
    out = []
    for batch in batches:
        rng = random.Random(batch)
        fr = lambda n: device_fr(rng, n)
        u64 = lambda n: device(struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)]))
        u32 = lambda n: device(struct.pack(f"<{n}I", *[rng.randrange(1 << depth) for _ in range(n)]))
        ins = [fr(batch), fr(batch), fr(batch), u64(batch), u32(batch), fr(batch), fr(batch), fr(depth * batch), u32(batch)]
        rs = fr(2 * batch)
        proofs = torch.empty(256 * batch, dtype=torch.uint8, device="cuda")
        pub = torch.empty(192 * batch, dtype=torch.uint8, device="cuda")
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
        out.append({"statement": "ragequit", "depth": depth, "batch": batch, "plan": PK.prover_plan(batch),
                    "ms_per_step": [round(t, 3) for t in times], "proofs_per_s": round(batch / (statistics.median(times) / 1e3), 1)})
        del ins, rs, proofs, pub
    PK.close()
    return out


def witness_kernels_ms(ctx, depth, batch):
    """k_ragequit_witness and k_owned_labeled_transfer_witness over `batch` proofs each in a launch of its own, alternated
    twice."""
    rng = random.Random(5)
    fr = lambda n: b"".join(rng.randrange(1 << 248).to_bytes(32, "little") for _ in range(n))
    u64 = lambda n: struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)])
    bits = lambda n: [rng.randrange(1 << depth) for _ in range(n)]
    labels = lambda n: [rng.randrange(1 << 32) for _ in range(n)]
    r_in = (fr(batch), fr(batch), fr(batch), u64(batch), labels(batch), fr(batch), fr(batch), fr(depth * batch), bits(batch))
    l_in = (fr(batch), fr(batch), fr(batch), u64(batch), labels(batch), fr(2 * batch), fr(2 * batch), u64(2 * batch),
            fr(2 * depth * batch), bits(2 * batch), fr(2 * batch), fr(2 * batch), u64(2 * batch), fr(depth * batch), bits(batch))
    calls = (("k_ragequit_witness", lambda: ctx.ragequit_witness(depth, *r_in)),
             ("k_owned_labeled_transfer_witness", lambda: ctx.owned_labeled_transfer_witness(depth, *l_in)))
    out = {name: [] for name, _ in calls}
    for name, call in calls:
        call()
    for _ in range(2):
        for name, call in calls:
            out[name].append(profile_step(ctx, call).get(name))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--depth", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ragequit: no CUDA device")
    info = gpu_info()
    for stmt in ("ragequit", "owned_labeled_transfer", "ragequit", "owned_labeled_transfer"):
        ctx = ob.Context(0)                # a context per pass: one prover's scratch lanes are released before the next's
        rate = prove_rate if stmt == "ragequit" else olt_prove_rate
        for r in rate(ctx, args.depth, args.batch, args.steps, args.warmup):
            print(json.dumps(dict(r, gpu=info)), flush=True)
        ctx.close()
    ctx = ob.Context(0)
    print(json.dumps({"witness_kernels_ms": witness_kernels_ms(ctx, args.depth, min(args.batch)), "batch": min(args.batch),
                      "depth": args.depth, "gpu": gpu_info()}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
