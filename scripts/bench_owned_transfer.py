#!/usr/bin/env python
"""Owned transfer proofs per second on one GPU, inputs resident in HBM (og_groth16_prove_owned_transfer_dev), next to transfer
proofs (og_groth16_prove_transfer_dev) measured in the same run on the same card, since the two statements share a domain and
differ by 4 % in size.

Per statement: a depth-32 key from the development setup; per batch `--warmup` untimed steps, then `--steps` timed steps,
each one call for the whole batch, timed with CUDA events on the library stream; the median step gives proofs/s.  Then:
  - k_owned_transfer_witness and k_transfer_witness over 1 024 proofs each in launches of their own (og_profile);
  - og_owned_note_scan_dev against og_note_scan_dev over 2^20 records x 8 keys (median of --steps after --warmup), the
    records being owned notes for the first and transfer notes for the second, 1 in 1 000 of them to one of the 8 wallets.
The card's name, power limit and SM clock (nvidia-smi, read only) are printed with the results.
Usage: python scripts/bench_owned_transfer.py [--batch 1024 4096] [--steps 5] [--warmup 2] [--depth 32]"""
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
from bench_transfer import device, device_fr, profile_step

R = ob.FR_MODULUS


def prove_rate(ctx, stmt, depth, batches, steps, warmup):
    """proofs/s of statement `stmt` ("transfer" or "owned_transfer") at each batch: random inputs of the eleven arrays (their
    proofs need not verify: the prover's work does not depend on it)."""
    rng = random.Random(7)
    setup = ob.setup_owned_transfer if stmt == "owned_transfer" else ob.setup_transfer
    PK = ob.ProvingKey(ctx, setup(ctx, depth, *[rng.randrange(1, R) for _ in range(5)])[0])
    fn = getattr(api.lib(), f"og_groth16_prove_{stmt}_dev")
    out = []
    for batch in batches:
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
        out.append({"statement": stmt, "depth": depth, "batch": batch, "plan": PK.prover_plan(batch),
                    "ms_per_step": [round(t, 3) for t in times], "proofs_per_s": round(batch / (statistics.median(times) / 1e3), 1)})
        del ins, rs, proofs, pub
    PK.close()
    return out


def witness_kernels_ms(ctx, depth, batch):
    """k_owned_transfer_witness and k_transfer_witness over `batch` proofs each in a launch of its own, with nothing else on
    the GPU, alternated twice."""
    rng = random.Random(5)
    fr = lambda n: b"".join(rng.randrange(1 << 248).to_bytes(32, "little") for _ in range(n))
    u64 = lambda n: struct.pack(f"<{n}Q", *[rng.randrange(1 << 64) for _ in range(n)])
    t_in = (fr(batch), fr(batch), fr(batch), fr(2 * batch), fr(2 * batch), u64(2 * batch), fr(2 * depth * batch),
            [rng.randrange(1 << depth) for _ in range(2 * batch)], fr(2 * batch), fr(2 * batch), u64(2 * batch))
    calls = (("k_owned_transfer_witness", lambda: ctx.owned_transfer_witness(depth, *t_in)),
             ("k_transfer_witness", lambda: ctx.transfer_witness(depth, *t_in)))
    out = {name: [] for name, _ in calls}
    for name, call in calls:
        call()
    for _ in range(2):
        for name, call in calls:
            out[name].append(profile_step(ctx, call).get(name))
    return out


def scan_ms(ctx, steps, warmup):
    """og_owned_note_scan_dev and og_note_scan_dev over 2^20 records x 8 keys."""
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
            to_dev(rng.integers(0, 1 << 63, size=n, dtype=np.uint64)), to_dev(eph)]
    recs = {k: (torch.empty(160 * n, dtype=torch.uint8, device=dev), torch.empty(32 * n, dtype=torch.uint8, device=dev))
            for k in ("owned", "plain")}
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    ctx.owned_note_encrypt_dev(*d_in, n, *recs["owned"], d_st)
    ctx.note_encrypt_dev(*d_in, n, *recs["plain"], d_st)
    d_owner = torch.empty(n, dtype=torch.int32, device=dev)
    d_plain = torch.empty(128 * n, dtype=torch.uint8, device=dev)
    ctx.sync()
    calls = {"og_owned_note_scan": lambda: ctx.owned_note_scan_dev(vb, sp, *recs["owned"], n, d_owner, d_plain),
             "og_note_scan": lambda: ctx.note_scan_dev(vb, *recs["plain"], n, d_owner, d_plain)}
    ms = {k: [] for k in calls}
    for _ in range(warmup):
        for call in calls.values():
            call()
    for _ in range(steps):                 # alternated, so both see the same clocks
        for k, call in calls.items():
            ctx.timer_start()
            call()
            ms[k].append(ctx.timer_stop())
    calls["og_owned_note_scan"]()
    ctx.sync()
    found = sum(1 for o in d_owner.cpu().tolist() if 0 <= o < 8)
    return {"records": n, "keys": 8, "owned_found": found, "expected_owned": int(mine.sum()),
            **{k: {"ms_median": round(statistics.median(v), 2), "ms": [round(x, 2) for x in v]} for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--depth", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_owned_transfer: no CUDA device")
    info = gpu_info()
    ctx = ob.Context(0)
    for stmt in ("owned_transfer", "transfer", "owned_transfer", "transfer"):
        for r in prove_rate(ctx, stmt, args.depth, args.batch, args.steps, args.warmup):
            print(json.dumps(dict(r, gpu=info)), flush=True)
    ctx.close()
    ctx = ob.Context(0)                    # a fresh context: the provers' scratch is released first
    print(json.dumps({"witness_kernels_ms": witness_kernels_ms(ctx, args.depth, min(args.batch)), "batch": min(args.batch),
                      "depth": args.depth, "gpu": info}), flush=True)
    print(json.dumps({"scan": scan_ms(ctx, args.steps, args.warmup), "gpu": gpu_info()}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
