#!/usr/bin/env python
"""Wall time of the setup ceremony's steps on one GPU: a phase-1 contribution and its verification at log_max 15, 16 and
20, and at each size the derivation of the largest circuit key that fits (the depth-32 withdraw key, domain 2^15, and the
depth-32 transfer key, domain 2^16) with one phase-2 contribution and its verification.  Prints one JSON line per step
with the card name and power limit read in the same run.
Usage: python scripts/bench_ceremony.py [--log-max 15 16 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import owshen_b200 as ob  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def timed(fn):
    t = time.perf_counter()
    r = fn()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-max", type=int, nargs="+", default=[15, 16, 20])
    args = ap.parse_args()
    name, power = card()
    ctx = ob.Context(0)
    ob.ptau_contribute(ctx, ob.ptau_new(ctx, 2))          # module load and generator tables outside the timings

    def out(step, log_max, s):
        print(json.dumps(dict(step=step, log_max=log_max, seconds=round(s, 3), card=name, power_limit=power)), flush=True)

    for lm in args.log_max:
        acc0 = ob.ptau_new(ctx, lm)
        (acc1, rec), s = timed(lambda: ob.ptau_contribute(ctx, acc0))
        out("ptau_contribute", lm, s)
        ok, s = timed(lambda: ob.ptau_verify(ctx, acc0, acc1, rec))
        assert ok
        out("ptau_verify", lm, s)
        if lm >= 16:
            (pk, vk), s = timed(lambda: ob.ptau_prepare_transfer(ctx, acc1, 32))
            out("ptau_prepare_transfer32", lm, s)
        else:
            (pk, vk), s = timed(lambda: ob.ptau_prepare_withdraw(ctx, acc1, 32))
            out("ptau_prepare_withdraw32", lm, s)
        (pk1, vk1, rec2), s = timed(lambda: ob.phase2_contribute(ctx, pk, vk))
        out("phase2_contribute", lm, s)
        ok, s = timed(lambda: ob.phase2_verify(ctx, pk, vk, pk1, vk1, rec2))
        assert ok
        out("phase2_verify", lm, s)
    ctx.close()


if __name__ == "__main__":
    main()
