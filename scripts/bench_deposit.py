#!/usr/bin/env python
"""Deposit proofs per second on one GPU, inputs resident in HBM (og_groth16_prove_deposit_dev).

Each configuration: a deposit key from the development setup, `--warmup` untimed steps, then `--steps` timed steps, each
one call for the whole batch, timed with CUDA events on the library stream.  One JSON line per (batch, window bits).
  --profile       also print a per-kernel split (og_profile) of one more step, which is not part of the timing
  --sweep         window bits of each MSM (A, B, C') at -2, -1, +1, +2 around the rule, the others at the rule
  --repeat N      run the list of configurations N times, alternating, so drifts in clock or load hit all of them
The GPU name and its power limit (nvidia-smi, read only) are printed with every line.
Usage: python scripts/bench_deposit.py [--batch 1024 16384] [--steps 5] [--warmup 2] [--profile] [--sweep] [--repeat 1]"""
import argparse
import json
import os
import random
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

import owshen_b200 as ob
from owshen_b200 import api

R = ob.FR_MODULUS
WINDOW_ENV = ("OG_C_A", "OG_C_B", "OG_C_C")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"gpu": out[0].strip(), "power_limit_w": float(out[1])}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}


def device_bytes(rng, n, bits=248):
    vals = [rng.randrange(1 << bits) for _ in range(n)]
    return torch.frombuffer(bytearray(b"".join(v.to_bytes(32, "little") for v in vals)), dtype=torch.uint8).to("cuda")


def run(ctx, pk_bytes, batch, steps, warmup, windows, profile):
    for name, c in zip(WINDOW_ENV, windows or (None,) * 3):
        if c is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = str(c)
    PK = ob.ProvingKey(ctx, pk_bytes)                     # window bits are read when the key is loaded
    rng = random.Random(batch)
    nul, sec, dep = (device_bytes(rng, batch) for _ in range(3))
    rs = device_bytes(rng, 2 * batch)
    proofs = torch.empty(256 * batch, dtype=torch.uint8, device="cuda")
    pub = torch.empty(64 * batch, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    L = api.lib()

    def step():
        rc = L.og_groth16_prove_deposit_dev(ctx._h, PK._h, nul.data_ptr(), sec.data_ptr(), dep.data_ptr(), batch, rs.data_ptr(),
                                            proofs.data_ptr(), pub.data_ptr())
        assert rc == 0, ob.OwshenB200Error(rc)

    for _ in range(warmup):
        step()
    ctx.sync()
    times = []
    for _ in range(steps):
        ctx.timer_start()
        step()
        times.append(ctx.timer_stop())
    out = {"batch": batch, "window_bits": list(PK.window_bits), "ms_per_step": [round(t, 3) for t in times],
           "proofs_per_s": round(batch / (sorted(times)[len(times) // 2] / 1e3), 1)}
    if profile:
        ctx.profile(True)
        step()
        ctx.sync()
        ctx.profile(False)
        prof = ctx.profile_dump()
        out["kernels_ms"] = {k: round(v[1], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][1])}
    PK.close()
    for name in WINDOW_ENV:
        os.environ.pop(name, None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[1024, 16384])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--repeat", type=int, default=1)
    args = ap.parse_args()
    ctx = ob.Context(0)
    rng = random.Random(7)
    pk, _ = ob.setup_deposit(ctx, *[rng.randrange(1, R) for _ in range(5)])
    PK = ob.ProvingKey(ctx, pk)
    rule = PK.window_bits
    PK.close()
    configs = [None]
    if args.sweep:
        for k in range(3):
            for d in (-2, -1, 1, 2):
                c = list(rule)
                c[k] += d
                if 2 <= c[k] <= 16:
                    configs.append(tuple(c))
    info = gpu_info()
    for _ in range(args.repeat):
        for batch in args.batch:
            for windows in configs:
                r = run(ctx, pk, batch, args.steps, args.warmup, windows, args.profile)
                r.update(info, rule=list(rule), steps=args.steps, warmup=args.warmup)
                print(json.dumps(r), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
