"""The prover's G2 and G1 MSMs inside the headline workload: 1024 depth-32 withdraw proofs per step (bench.py's step), per-kernel
CUDA-event times from og_profile for the G2 and G1 bucket accumulations, their reductions and heavy buckets, and the whole step.

The G2 accumulation's share of the carry-chain peak is computed from static counts: one mixed addition per (point, window)
of the B MSM and WIDE_PER_MADD 32x32->64 multiply-adds per addition (8 lazy Fq2 products of 3 wide products + 2 reductions =
320, 2 lazy Fq2 squarings of 2 wide products + 2 reductions = 256: fp.cuh), against og_int_pipe_peaks measured in the same
run.  The G1 accumulation's share is computed over the A and C' MSMs from the expected number of mixed additions under uniform
digits -- per (proof, window) the nonzero digits minus the occupied buckets, since the first point of a bucket is stored, not
added; about 0.56 of bench.py's one addition per (point, window) -- with G1_WIDE_PER_MADD multiply-adds per addition: 6 lazy
products of 128 (interleaved Montgomery), the one-reduction Y3 of 192 (two products and one reduction, mont_mul_sum_lazy) and
2 lazy squarings of 36 + 64, 1160 in all (fp.cuh).  Builds before the lazy G1 accumulation spent 1224 (8 x 128 + 2 x 100);
--g1-wide-per-madd 1224 reports an older library's share.  The card's name, power limit and SM clock are read with read-only
nvidia-smi queries in the same call.

OWSHEN_B200_LIB=<path> runs another build of the library, so that two builds can be alternated in one session:
    for i in 1 2 3; do OWSHEN_B200_LIB=old.so python scripts/bench_g2_msm.py; python scripts/bench_g2_msm.py; done
Usage: python scripts/bench_g2_msm.py [--steps 3] [--warmup 2] [--batch 1024] [--g1-wide-per-madd 1160]"""
import argparse
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WIDE_PER_MADD = 8 * 320 + 2 * 256
G1_WIDE_PER_MADD = 6 * 128 + 192 + 2 * (36 + 64)
KERNELS = ("k_bucket_acc_g2", "k_reduce_level_g2", "k_bucket_heavy_g2", "k_bucket_acc_g1", "k_reduce_level_g1")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl, sm, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_mhz_now": float(sm), "sm_max_mhz": float(smax)}
    except Exception as e:  # the numbers are still reported; the card is then unknown
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--g1-wide-per-madd", type=int, default=G1_WIDE_PER_MADD)
    args = ap.parse_args()

    import torch
    import bench
    import owshen_b200 as ob
    from owshen_b200 import api

    if not torch.cuda.is_available():
        sys.exit("bench_g2_msm: no CUDA device")
    dev = torch.device("cuda", 0)
    ctx = ob.Context(0)
    pk_bytes, _ = ob.setup_withdraw(ctx, bench.DEPTH, *bench.toxic(random.Random(bench.TOXIC_SEED)))
    PK = ob.ProvingKey(ctx, pk_bytes)
    nul, sec, rec, sib, bits, rs = bench.synth_inputs(random.Random(4096), args.batch, bench.DEPTH)
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8).to(dev)
    d_nul, d_sec, d_rec, d_sib, d_rs = (u8(x) for x in (nul, sec, rec, sib, rs))
    d_bits = torch.tensor([b if b < 2**31 else b - 2**32 for b in bits], dtype=torch.int32, device=dev)
    d_proofs = torch.empty(256 * args.batch, dtype=torch.uint8, device=dev)
    d_pub = torch.empty(96 * args.batch, dtype=torch.uint8, device=dev)
    L = api.lib()

    def step():
        rc = L.og_groth16_prove_withdraw_dev(ctx._h, PK._h, d_nul.data_ptr(), d_sec.data_ptr(), d_rec.data_ptr(), d_sib.data_ptr(),
                                             d_bits.data_ptr(), args.batch, d_rs.data_ptr(), d_proofs.data_ptr(), d_pub.data_ptr())
        if rc:
            raise ob.OwshenB200Error(rc, L.og_last_error(ctx._h).decode())

    for _ in range(args.warmup):
        step()
    ctx.sync()
    sampler = bench.ClockSampler(0)
    sampler.start()
    ctx.timer_start()
    for _ in range(args.steps):
        step()
    step_ms = ctx.timer_stop() / args.steps
    ctx.sync()
    clocks = sampler.stop()
    ctx.profile(True)                       # per-kernel times in a run of their own: the events slow the step a little
    for _ in range(args.steps):
        step()
    ctx.sync()
    ctx.profile(False)
    prof = ctx.profile_dump()
    pipes = ctx.int_pipe_peaks()

    c_b = PK.window_bits[1]
    n_b = 12294                             # points of the B MSM of the depth-32 withdraw key (DESIGN.md section 5.5)
    madds = args.batch * n_b * ((255 + c_b - 1) // c_b)
    peak = pipes["imad_wide_carry_chain_per_s"]
    floor_ms = 1e3 * madds * WIDE_PER_MADD / peak
    per_step = {k: prof[k][1] / args.steps for k in KERNELS if k in prof}
    acc = per_step.get("k_bucket_acc_g2")
    # G1: one mixed addition per (point, window) of the A and C' MSMs, as bench.py counts them
    info = api.r1cs_info(bench.DEPTH)
    m = 1 << info["log_m"]
    n_supp = len(set(api.r1cs_export(bench.DEPTH, "B")[1]))
    n_priv = info["n_vars"] - info["n_pub"] - 1
    win = lambda c: (255 + c - 1) // c
    c_a, c_c = PK.window_bits[0], PK.window_bits[2]
    def adds(n, c):                         # expected mixed additions of one (proof, window) group: entries - occupied buckets
        nb, k = 1 << (c - 1), n * (1 - 2.0 ** -c)
        return k - nb * (1 - (1 - 1 / nb) ** k)
    g1_madds = args.batch * (adds(info["n_vars"] + 2, c_a) * win(c_a) + adds(n_priv + n_supp + m + 1, c_c) * win(c_c))
    g1_floor_ms = 1e3 * g1_madds * args.g1_wide_per_madd / peak
    acc1 = per_step.get("k_bucket_acc_g1")
    out = {
        "lib": os.environ.get("OWSHEN_B200_LIB") or "in-tree",
        "gpu": gpu_info(), "sm_clock_timed": clocks,
        "step_ms": round(step_ms, 2), "proofs_per_s": round(args.batch / step_ms * 1e3, 1),
        "kernel_ms_per_step": {k: round(v, 2) for k, v in per_step.items()},
        "g2_madds_per_step": madds, "wide_madds_per_g2_madd": WIDE_PER_MADD,
        "carry_chain_peak_per_s": peak, "g2_acc_ms_at_peak": round(floor_ms, 1),
        "g2_acc_share_of_peak": round(floor_ms / acc, 3) if acc else None,
        "g1_madds_per_step": round(g1_madds), "wide_madds_per_g1_madd": args.g1_wide_per_madd, "g1_acc_ms_at_peak": round(g1_floor_ms, 1),
        "g1_acc_share_of_peak": round(g1_floor_ms / acc1, 3) if acc1 else None,
    }
    print(json.dumps(out))
    PK.close()
    ctx.close()


if __name__ == "__main__":
    main()
