#!/usr/bin/env python
"""Exclusion withdraw proofs per second on one GPU, inputs resident in HBM (og_groth16_prove_exclusion_dev).

A depth-32 exclusion key from the development setup; per batch `--warmup` untimed steps, then `--steps` timed steps, each one
call for the whole batch, timed with CUDA events on the library stream; the median step gives proofs/s.  One JSON line per
batch, with the key's window bits and prover plan (chunk, lanes, scratch per lane).
  --profile       also print a per-kernel split (og_profile) of one more step, which is not part of the timing,
                  k_exclusion_witness against k_withdraw_witness at the smallest batch, each in a launch of its own
                  (og_exclusion_witness / og_withdraw_witness, no lane overlap), and the time to build an ExclusionSet
                  (leaves in one og_mimc7_hash2 call, tree in one MerkleTree.insert_batch, host store included) over
                  --set-sizes flagged indices
The GPU name and its power limit (nvidia-smi, read only) are printed with every line.
Usage: python scripts/bench_exclusion.py [--batch 1024 4096] [--steps 5] [--warmup 2] [--profile] [--depth 32]
                                         [--set-sizes 65536 1048576]"""
import argparse
import json
import os
import random
import struct
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

import owshen_b200 as ob
from owshen_b200 import api
from scripts.bench_transfer import device, device_fr, gpu_info, profile_step

R = ob.FR_MODULUS


def run(ctx, PK, depth, batch, steps, warmup, profile):
    """Random notes, paths and keys (their proofs need not verify: the prover's work does not depend on it)."""
    rng = random.Random(batch)
    words = lambda n: device(struct.pack(f"<{n}I", *[rng.randrange(1 << depth) for _ in range(n)]))
    keys = lambda n: device(struct.pack(f"<{n}Q", *[rng.randrange(1 << 33) for _ in range(n)]))
    ins = [device_fr(rng, batch), device_fr(rng, batch), device_fr(rng, batch), device_fr(rng, depth * batch), words(batch),
           keys(batch), keys(batch), device_fr(rng, depth * batch), words(batch)]
    rs = device_fr(rng, 2 * batch)
    proofs = torch.empty(256 * batch, dtype=torch.uint8, device="cuda")
    pub = torch.empty(128 * batch, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    L = api.lib()

    def step():
        rc = L.og_groth16_prove_exclusion_dev(ctx._h, PK._h, *[t.data_ptr() for t in ins], batch, rs.data_ptr(), proofs.data_ptr(),
                                              pub.data_ptr())
        assert rc == 0, ob.OwshenB200Error(rc)

    for _ in range(warmup):
        step()
    ctx.sync()
    times = []
    for _ in range(steps):
        ctx.timer_start()
        step()
        times.append(ctx.timer_stop())
    out = {"depth": depth, "batch": batch, "window_bits": list(PK.window_bits), "plan": PK.prover_plan(batch),
           "ms_per_step": [round(t, 3) for t in times], "proofs_per_s": round(batch / (sorted(times)[len(times) // 2] / 1e3), 1)}
    if profile:
        out["kernels_ms"] = profile_step(ctx, step)
    return out


def witness_kernels_alone_ms(ctx, depth, batch):
    """k_exclusion_witness and k_withdraw_witness over `batch` proofs each in a launch of its own, with nothing else on the
    GPU: the two witness kernels compared without the prover's lane overlap."""
    rng = random.Random(5)
    fr = lambda n: b"".join(rng.randrange(1 << 248).to_bytes(32, "little") for _ in range(n))
    bits = lambda: [rng.randrange(1 << depth) for _ in range(batch)]
    keys = lambda: [rng.randrange(1 << 33) for _ in range(batch)]
    x_in = (fr(batch), fr(batch), fr(batch), fr(depth * batch), bits(), keys(), keys(), fr(depth * batch), bits())
    w_in = x_in[:5]
    out = {}
    for name, call in (("k_exclusion_witness", lambda: ctx.exclusion_witness(depth, *x_in)),
                       ("k_withdraw_witness", lambda: ctx.withdraw_witness(depth, *w_in))):
        call()
        out[name] = profile_step(ctx, call).get(name)
    return out


def exclusion_set_build_s(ctx, depth, n):
    """Wall time of ExclusionSet(ctx, depth, n random flagged indices), GPU hashing and the host-side store together."""
    rng = random.Random(n)
    flagged = rng.sample(range(1 << depth), n)
    ob.ExclusionSet(ctx, depth, flagged[:16])          # warm: module load, constants
    ctx.sync()
    t0 = time.perf_counter()
    xs = ob.ExclusionSet(ctx, depth, flagged)
    ctx.sync()
    return {"flagged": n, "seconds": round(time.perf_counter() - t0, 3), "leaves": len(xs) + 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--set-sizes", type=int, nargs="*", default=[1 << 16, 1 << 20])
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    ctx = ob.Context(0)
    rng = random.Random(7)
    pk, _ = ob.setup_exclusion(ctx, args.depth, *[rng.randrange(1, R) for _ in range(5)])
    PK = ob.ProvingKey(ctx, pk)
    info = gpu_info()
    results = [run(ctx, PK, args.depth, batch, args.steps, args.warmup, args.profile) for batch in args.batch]
    PK.close()
    ctx.close()
    if args.profile:
        ctx = ob.Context(0)     # a fresh context: the proving steps' scratch is released first
        alone = witness_kernels_alone_ms(ctx, args.depth, min(args.batch))
        sets = [exclusion_set_build_s(ctx, args.depth, n) for n in args.set_sizes]
        ctx.close()
        print(json.dumps({"witness_kernels_alone_ms": alone, "batch": min(args.batch), "depth": args.depth,
                          "exclusion_set_build": sets, **info}), flush=True)
    for r in results:
        r.update(info, steps=args.steps, warmup=args.warmup)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
