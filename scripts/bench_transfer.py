#!/usr/bin/env python
"""Transfer proofs per second on one GPU, inputs resident in HBM (og_groth16_prove_transfer_dev).

A depth-32 transfer key from the development setup; per batch `--warmup` untimed steps, then `--steps` timed steps, each one
call for the whole batch, timed with CUDA events on the library stream; the median step gives proofs/s.  One JSON line per
batch, with the key's window bits and prover plan (chunk, lanes, scratch per lane).
  --profile       also print a per-kernel split (og_profile) of one more step, which is not part of the timing, the
                  k_withdraw_witness time of one depth-32 withdraw step at the same batch next to k_transfer_witness, and
                  both witness kernels at the smallest batch in launches of their own (no lane overlap)
The GPU name and its power limit (nvidia-smi, read only) are printed with every line.
Usage: python scripts/bench_transfer.py [--batch 1024 4096] [--steps 5] [--warmup 2] [--profile] [--depth 32]"""
import argparse
import json
import os
import random
import struct
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

import owshen_b200 as ob
from owshen_b200 import api

R = ob.FR_MODULUS


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}


def device(b: bytes):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to("cuda")


def device_fr(rng, n, bits=248):
    return device(b"".join(rng.randrange(1 << bits).to_bytes(32, "little") for _ in range(n)))


def profile_step(ctx, step):
    ctx.profile(True)
    step()
    ctx.sync()
    ctx.profile(False)
    prof = ctx.profile_dump()
    return {k: round(v[1], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][1])}


def run(ctx, PK, depth, batch, steps, warmup, profile):
    """Random notes (their proofs need not verify: the prover's work does not depend on it)."""
    rng = random.Random(batch)
    fr = lambda n: device_fr(rng, n)
    u64 = lambda n: device(struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)]))
    ins = [fr(batch), fr(batch), fr(batch), fr(2 * batch), fr(2 * batch), u64(2 * batch), fr(2 * depth * batch),
           device(struct.pack(f"<{2 * batch}I", *[rng.randrange(1 << depth) for _ in range(2 * batch)])),
           fr(2 * batch), fr(2 * batch), u64(2 * batch)]
    rs = fr(2 * batch)
    proofs = torch.empty(256 * batch, dtype=torch.uint8, device="cuda")
    pub = torch.empty(256 * batch, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    L = api.lib()

    def step():
        rc = L.og_groth16_prove_transfer_dev(ctx._h, PK._h, *[t.data_ptr() for t in ins], batch, rs.data_ptr(), proofs.data_ptr(),
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


def withdraw_witness_ms(ctx, depth, batch):
    """k_withdraw_witness of one depth-`depth` withdraw step at `batch` proofs (og_profile), for comparison."""
    rng = random.Random(3)
    pk, _ = ob.setup_withdraw(ctx, depth, *[rng.randrange(1, R) for _ in range(5)])
    PK = ob.ProvingKey(ctx, pk)
    d = [device_fr(rng, batch) for _ in range(3)] + [device_fr(rng, batch * depth)]
    bits = device(struct.pack(f"<{batch}I", *[rng.randrange(1 << depth) for _ in range(batch)]))
    rs = device_fr(rng, 2 * batch)
    proofs = torch.empty(256 * batch, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def step():
        rc = api.lib().og_groth16_prove_withdraw_dev(ctx._h, PK._h, *[t.data_ptr() for t in d], bits.data_ptr(), batch,
                                                     rs.data_ptr(), proofs.data_ptr(), None)
        assert rc == 0, ob.OwshenB200Error(rc)

    step()
    ctx.sync()
    ms = profile_step(ctx, step).get("k_withdraw_witness")
    PK.close()
    return ms


def witness_kernels_alone_ms(ctx, depth, batch):
    """k_transfer_witness and k_withdraw_witness over `batch` proofs each in a launch of its own (og_transfer_witness /
    og_withdraw_witness), with nothing else on the GPU: the two witness kernels compared without the prover's lane overlap."""
    rng = random.Random(5)
    fr = lambda n: b"".join(rng.randrange(1 << 248).to_bytes(32, "little") for _ in range(n))
    u64 = lambda n: struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)])
    t_in = (fr(batch), fr(batch), fr(batch), fr(2 * batch), fr(2 * batch), u64(2 * batch), fr(2 * depth * batch),
            [rng.randrange(1 << depth) for _ in range(2 * batch)], fr(2 * batch), fr(2 * batch), u64(2 * batch))
    w_in = (fr(batch), fr(batch), fr(batch), fr(depth * batch), [rng.randrange(1 << depth) for _ in range(batch)])
    out = {}
    for name, call in (("k_transfer_witness", lambda: ctx.transfer_witness(depth, *t_in)),
                       ("k_withdraw_witness", lambda: ctx.withdraw_witness(depth, *w_in))):
        call()
        out[name] = profile_step(ctx, call).get(name)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    ctx = ob.Context(0)
    rng = random.Random(7)
    pk, _ = ob.setup_transfer(ctx, args.depth, *[rng.randrange(1, R) for _ in range(5)])
    PK = ob.ProvingKey(ctx, pk)
    info = gpu_info()
    results = [run(ctx, PK, args.depth, batch, args.steps, args.warmup, args.profile) for batch in args.batch]
    PK.close()
    ctx.close()
    if args.profile:
        ctx = ob.Context(0)     # a fresh context: the transfer steps' scratch is released first
        for r in results:
            r["k_withdraw_witness_ms_same_batch"] = withdraw_witness_ms(ctx, args.depth, r["batch"])
        alone = witness_kernels_alone_ms(ctx, args.depth, min(args.batch))
        ctx.close()
        print(json.dumps({"witness_kernels_alone_ms": alone, "batch": min(args.batch), "depth": args.depth}), flush=True)
    for r in results:
        r.update(info, steps=args.steps, warmup=args.warmup)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
