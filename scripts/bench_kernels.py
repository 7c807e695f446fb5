#!/usr/bin/env python
"""Per-kernel measurements for the BASELINE configs that are not the headline (which bench.py covers):
  config 2  batched MiMC7 Merkle paths, 4096 leaves x depth 32
  config 3  2^20-point G1 Pippenger MSM (uniform and witness-like scalars), plus a 2^18 G2 MSM
  NTT       2^20 forward, and the prover's shape (3072 x 2^15)
Inputs are resident in HBM (the `_dev` C-ABI entry points), timing is CUDA events on the library stream,
W warm-ups then K timed repetitions; inputs exceed or are re-generated so L2 does not serve them warm
(each repetition streams more scratch than the 50 MB L2 holds through L2 for the MSM/NTT; config 2 flushes explicitly).
Every line reports the algorithmic HBM fraction SURVEY.md section 8d asks for AND the integer-pipe
fraction (32x32->64 multiply-adds per second against og_int_pipe_peaks), which is the bound that binds.
Usage: python scripts/bench_kernels.py [--reps K] > kernels.jsonl
"""
import argparse
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import owshen_b200 as ob  # noqa: E402
from owshen_b200 import api  # noqa: E402

R = api.FR_MODULUS
WIDE_PER_MUL = 128          # 32x32->64 products per 256-bit Montgomery multiplication (64 a*b + 64 q*p)


def hbm_peak():
    try:
        return float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"]), "measured"
    except Exception:
        return 3350.0, "nominal"      # H100 SXM data sheet (HBM3)


def fr_bytes(rng, n):
    """n 248-bit values (always canonical), fast in bulk: inputs whose distribution does not matter (hash inputs, NTT data)."""
    raw = rng.randbytes(31 * n)
    return b"".join(raw[31 * i:31 * i + 31] + b"\0" for i in range(n))


def fr_uniform(rng, n):
    """n scalars uniform in [0, r) (SURVEY.md 8d: "uniform 254-bit"): 254 random bits, rejected above the modulus.  The
    248-bit generator above leaves the top window of an MSM with 8-bit digits -> 128 heavy buckets, which is not the workload."""
    out = bytearray()
    while len(out) < 32 * n:
        v = rng.getrandbits(254)
        if v < R:
            out += v.to_bytes(32, "little")
    return bytes(out)


def dev(b, device):
    return torch.frombuffer(bytearray(b), dtype=torch.uint8).to(device)


def timed(ctx, fn, warm, reps, flush=None):
    for _ in range(warm):
        fn()
    ctx.sync()
    tot = 0.0
    for _ in range(reps):
        if flush is not None:
            flush.add_(1)
            torch.cuda.synchronize()
        ctx.timer_start()
        fn()
        tot += ctx.timer_stop()
    return tot / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    device = torch.device("cuda", 0)
    ctx = ob.Context(0)
    L = api.lib()
    rng = random.Random(3)
    peak, peak_src = hbm_peak()
    pipes = ctx.int_pipe_peaks()
    print(json.dumps({"kernel": "int_pipe_peaks", **pipes, "note": "multiply-adds per second; carry-chain figure is the Montgomery-row shape"}), flush=True)
    print(json.dumps({"kernel": "fp64_peak", "dfma_per_s": ctx.fp64_peak(), "note": "FP64 pipe is idle in every kernel of this library (planning probe)"}), flush=True)
    print(json.dumps({"kernel": "hybrid_probe", **ctx.hybrid_probe(),
                      "note": "52x52-bit products on the FP64 pipe vs 32x32-bit carry-chain IMAD.WIDE, alone and interleaved (round-2 planning)"}), flush=True)
    wide_peak = pipes["imad_wide_carry_chain_per_s"]
    flush = torch.zeros(256 << 20, dtype=torch.uint8, device=device)    # 256 MB > L2

    def check(rc):
        if rc != 0:
            raise ob.OwshenB200Error(rc, L.og_last_error(ctx._h).decode())

    def line(name, ms, alg_bytes, muls, extra):
        gbs = alg_bytes / (ms * 1e-3) / 1e9
        wide = muls * WIDE_PER_MUL / (ms * 1e-3)
        print(json.dumps({"kernel": name, "ms": ms, "algorithmic_bytes": alg_bytes, "hbm_gbs": gbs, "hbm_frac": gbs / peak,
                          "hbm_peak": peak, "hbm_peak_source": peak_src, "field_muls": muls, "wide_mad_per_s": wide,
                          "int_pipe_frac": wide / wide_peak, **extra}), flush=True)

    # ---- config 2 -------------------------------------------------------------------------------
    n, depth = 4096, 32
    leaves, sib = dev(fr_bytes(rng, n), device), dev(fr_bytes(rng, n * depth), device)
    bits = torch.tensor([rng.randrange(1 << 31) for _ in range(n)], dtype=torch.int32, device=device)
    out = torch.empty(32 * n * (depth + 1), dtype=torch.uint8, device=device)
    torch.cuda.synchronize()
    ms = timed(ctx, lambda: check(L.og_mimc7_merkle_paths_dev(ctx._h, leaves.data_ptr(), sib.data_ptr(), bits.data_ptr(), n, depth, out.data_ptr())),
               args.warmup, args.reps, flush)
    alg = n * (32 + 32 * depth + 4) + n * (depth + 1) * 32
    line("mimc7_merkle_paths_4096x32 (config 2)", ms, alg, n * depth * 2 * 91 * 4,
         {"hashes_per_s": n * depth / (ms * 1e-3), "l2": "256 MB flush between repetitions"})

    # ---- config 3 -------------------------------------------------------------------------------
    for log_n, curve in ((20, "g1"), (18, "g2")):
        n = 1 << log_n
        sc_pts = fr_bytes(rng, n)
        pts_host = ctx.g1_generator_mul(sc_pts) if curve == "g1" else ctx.g2_generator_mul(sc_pts)
        pts = dev(pts_host, device)
        outp = torch.empty(64 if curve == "g1" else 128, dtype=torch.uint8, device=device)
        fn_ = L.og_msm_g1_dev if curve == "g1" else L.og_msm_g2_dev
        kinds = {"uniform": fr_uniform(rng, n)}
        if curve == "g1":
            wl = bytearray(fr_uniform(rng, n))
            for i in range(n):
                u = rng.random()
                if u < 0.6:
                    wl[32 * i:32 * i + 32] = (rng.randrange(2)).to_bytes(32, "little")
                elif u < 0.9:
                    wl[32 * i + 8:32 * i + 32] = bytes(24)
            kinds["witness-like"] = bytes(wl)
        for kind, sc in kinds.items():
            scd = dev(sc, device)
            torch.cuda.synchronize()
            ms = timed(ctx, lambda: check(fn_(ctx._h, pts.data_ptr(), scd.data_ptr(), n, outp.data_ptr())), args.warmup, args.reps)
            ctx.profile(True)
            check(fn_(ctx._h, pts.data_ptr(), scd.data_ptr(), n, outp.data_ptr()))
            prof = ctx.profile_dump()
            ctx.profile(False)
            per_pair = 96 if curve == "g1" else 160
            c = min(16, max(2, log_n - 3)); windows = (255 + c - 1) // c
            madds = n * windows if kind == "uniform" else None
            muls = (madds * (10 if curve == "g1" else 28)) if madds else 0
            line(f"msm_{curve}_2^{log_n}_{kind} (config 3)", ms, per_pair * n, muls,
                 {"points_per_s": n / (ms * 1e-3), "window_bits": c, "windows": windows,
                  "kernels_ms_one_run": {k: round(v[1], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][1])[:8]},
                  "l2": "sorted digit lists + buckets (> 50 MB) stream through L2 every repetition"})

    # ---- NTT ------------------------------------------------------------------------------------
    for log_n, batch in ((20, 1), (15, 3072), (24, 1)):
        n = 1 << log_n
        data = torch.randint(0, 255, (32 * n * batch,), dtype=torch.uint8, device=device)
        data.view(-1, 32)[:, 31] = 0                      # canonical (< 2^248)
        torch.cuda.synchronize()
        ms = timed(ctx, lambda: check(L.og_ntt_dev(ctx._h, data.data_ptr(), log_n, batch, 0, 0)), args.warmup, args.reps,
                   flush if n * batch * 32 < (200 << 20) else None)
        line(f"ntt_2^{log_n}_x{batch} (bytes in/out incl. Montgomery conversion kernels)", ms, 64 * n * batch, int(n * batch * (log_n / 2 + 2 - 0.75)),
             {"elements_per_s": n * batch / (ms * 1e-3), "note": "products counted: n/2*log n butterflies - 0.75 n skipped unit twiddles + 2 n boundary conversions"})
    # ---- BabyJubJub batch signing and verification (SURVEY 8f.3): device-resident, CUDA-event timed -------------------
    n = 1 << 16
    sk, rnd, msg = (dev(fr_bytes(rng, n), device) for _ in range(3))
    pkx = torch.empty(32 * n, dtype=torch.uint8, device=device); odd = torch.empty(n, dtype=torch.uint8, device=device)
    sg = torch.empty(96 * n, dtype=torch.uint8, device=device); st = torch.empty(n, dtype=torch.uint8, device=device)
    torch.cuda.synchronize()
    for hk in (0, 1):
        ms = timed(ctx, lambda: check(L.og_bjj_sign_batch_dev(ctx._h, sk.data_ptr(), rnd.data_ptr(), msg.data_ptr(), n, hk, pkx.data_ptr(), odd.data_ptr(),
                                                             sg.data_ptr(), st.data_ptr())), args.warmup, args.reps)
        # 2 fixed-base multiplications through the window table (64 additions x ~14 products) + 2 inversions (~380) + the hash
        muls = n * (2 * 64 * 14 + 2 * 380 + (7 * 364 if hk else 5))
        line(f"bjj_sign_batch_65536 hash_kind={hk} (to_pub + sign, mod.rs:206-237)", ms, n * (96 + 32 + 1 + 96 + 1), muls,
             {"signatures_per_s": n / (ms * 1e-3), "signed": int((st == 1).sum().item())})
        ms = timed(ctx, lambda: check(L.og_bjj_verify_batch_dev(ctx._h, pkx.data_ptr(), odd.data_ptr(), msg.data_ptr(), sg.data_ptr(), n, hk, st.data_ptr())),
                   args.warmup, args.reps)
        # decompress (one inversion + a square root: ~4 x 380 products) + h * A (256 doublings x 8 + ~128 additions x 14) + s * BASE (table)
        muls = n * (4 * 380 + 256 * 8 + 128 * 14 + 64 * 14 + (5 * 364 if hk else 4))
        line(f"bjj_verify_batch_65536 hash_kind={hk} (valid signatures from the line above)", ms, n * (32 + 1 + 32 + 96 + 1), muls,
             {"signatures_per_s": n / (ms * 1e-3), "verified": int((st == 1).sum().item())})
    ctx.close()


if __name__ == "__main__":
    main()
