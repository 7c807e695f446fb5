"""Encrypted notes on the GPU: encryption and scanning rates with inputs resident in HBM (the `_dev` entry points), timed with
CUDA events on the library's stream, median of --steps after --warmup; a per-kernel split from og_profile in a separate run;
the scan's share of the carry-chain peak from the operation count below and og_int_pipe_peaks measured in the same run; the
card's name and power limit from read-only nvidia-smi queries.

Operation count of one (record, key) pair in k_note_scan, in Fr products (one product = 64 + 64 = 128 carry-chain 32x32-bit
multiply-adds: the 8x8-limb product and its Montgomery reduction):
  v E' by the 4-bit window: 252 doublings x 8 + at most 78 additions x 13 = 3030
  affine(S): one inversion by exponentiation, about 256 squarings + 128 products, and 2 products = 386
  MiMC7: k (2 permutations) and the 4 pads, 6 x 91 rounds x 4 products = 2184 (a foreign record stops there: its amount
  is not below 2^64, so the 4 permutations of the commitment run only for candidate notes)
Usage: python scripts/bench_notes.py [--steps 5] [--warmup 2]"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

PRODUCTS_PER_PAIR = 3030 + 386 + 2184
MADDS_PER_PRODUCT = 128


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import numpy as np
    import torch
    import owshen_b200 as ob
    from bench_g2_msm import gpu_info

    if not torch.cuda.is_available():
        sys.exit("bench_notes: no CUDA device")
    dev = torch.device("cuda", 0)
    ctx = ob.Context(0)
    rng = np.random.default_rng(2026)
    nmax = 1 << 20
    keys = [int.from_bytes(rng.integers(0, 256, 31, dtype=np.uint8).tobytes(), "little") + 1 for _ in range(8)]
    kb = b"".join(k.to_bytes(32, "little") for k in keys)
    foreign = b"".join((int.from_bytes(rng.integers(0, 256, 31, dtype=np.uint8).tobytes(), "little") + 1).to_bytes(32, "little")
                       for _ in range(64))
    px, odd = ctx.note_public_keys(kb + foreign)
    px = np.frombuffer(px, dtype=np.uint8).reshape(72, 32)
    odd = np.frombuffer(odd, dtype=np.uint8)
    dest = rng.integers(8, 72, size=nmax)
    dest[rng.choice(nmax, size=nmax // 1000, replace=False)] = rng.integers(0, 8, size=nmax // 1000)

    def rand_fr(top_bits):
        a = rng.integers(0, 256, size=(nmax, 32), dtype=np.uint8)
        a[:, 31] &= (1 << top_bits) - 1
        return a

    eph = rand_fr(2)
    eph[:, 0] |= 1
    to_dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).reshape(-1).view(np.uint8)).to(dev)
    d_in = [to_dev(px[dest]), to_dev(odd[dest]), to_dev(rand_fr(5)), to_dev(rand_fr(5)), to_dev(rand_fr(5)),
            to_dev(rng.integers(0, 1 << 63, size=nmax, dtype=np.uint64)), to_dev(eph)]
    d_rec = torch.empty(160 * nmax, dtype=torch.uint8, device=dev)
    d_cm = torch.empty(32 * nmax, dtype=torch.uint8, device=dev)
    d_st = torch.empty(nmax, dtype=torch.uint8, device=dev)
    d_owner = torch.empty(nmax, dtype=torch.int32, device=dev)
    d_plain = torch.empty(128 * nmax, dtype=torch.uint8, device=dev)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        ms = []
        for _ in range(args.steps):
            ctx.timer_start()
            fn()
            ms.append(ctx.timer_stop())
        return statistics.median(ms), min(ms), max(ms)

    peaks = ctx.int_pipe_peaks()
    chain_peak = peaks["imad_wide_carry_chain_per_s"]
    results = {"gpu": gpu_info(), "int_pipe_peaks": peaks, "steps": args.steps, "warmup": args.warmup, "encrypt": [], "scan": []}
    encrypt = lambda n: ctx.note_encrypt_dev(*d_in, n, d_rec, d_cm, d_st)
    for n in (1 << 16, 1 << 20):
        med, lo, hi = timed(lambda: encrypt(n))
        results["encrypt"].append({"n": n, "ms": med, "ms_min": lo, "ms_max": hi, "notes_per_s": n / med * 1e3})
    encrypt(nmax)
    ctx.sync()
    assert bytes(d_st.cpu().numpy()) == b"\x01" * nmax
    for n in (1 << 16, 1 << 20):
        for k in (1, 8):
            med, lo, hi = timed(lambda: ctx.note_scan_dev(kb[:32 * k], d_rec, d_cm, n, d_owner, d_plain))
            pairs = n * k / med * 1e3
            results["scan"].append({"n": n, "keys": k, "ms": med, "ms_min": lo, "ms_max": hi, "records_per_s": n / med * 1e3,
                                    "pairs_per_s": pairs, "share_of_carry_chain_peak": pairs * PRODUCTS_PER_PAIR * MADDS_PER_PRODUCT / chain_peak})
    # per-kernel split of one 2^20 x 8 scan and one 2^20 encryption, in a separate profiled run
    ctx.profile(True)
    ctx.note_scan_dev(kb, d_rec, d_cm, nmax, d_owner, d_plain)
    encrypt(nmax)
    results["profile"] = ctx.profile_dump()
    ctx.profile(False)
    found = int((d_owner != -1).sum().item())
    results["owned_in_last_scan"] = found
    print(json.dumps(results, indent=1))
    ctx.close()


if __name__ == "__main__":
    main()
