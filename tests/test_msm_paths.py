"""The one-shot MSM engine (msm.cu) at every window size, reduction path, heavy-bucket path and runtime knob, against the
oracle; and the batched prover at non-default window bits.

A one-shot MSM is a family of code paths: the window size c follows the input size (pick_window), G1 inputs of 1024 or more
points go through GLV (2n points, 127-bit scalars), the reduction above level 0 switches to the tree-sum tail when enough bucket
sums remain (cut into 1, 2, 4 or 8 slices), overfull buckets go to the segmented heavy-bucket kernels, and OG_GLV, OG_MSM_TAIL
and OG_RED_FAN0 move the boundaries.  `msm_path` below restates that selection in Python.  A CPU test checks that the sweep
table built from it reaches every path; the GPU tests compare every case with the oracle byte for byte and check, through the
library's per-kernel profile, that the kernels the mirror predicts are the ones that ran, so the mirror cannot drift from msm.cu.

Reference values: points are generated as known multiples d_i G (og_*_generator_mul, itself checked against the oracle), so
sum k_i P_i = (sum k_i d_i mod r) G is one fixed-base multiplication by the oracle's C port, exact at any size.  Inputs small
enough for the oracle's CPU MSM are compared with cport.g1_msm / cport.g2_msm as well."""
import os
import random

import pytest

import owshen_b200 as ob
from oracle import bn254 as bn
from oracle import cport
from tests.helpers import rand_inputs, withdraw_keys32
from tests.test_host_limbs import h      # noqa: F401  (host harness fixture: glv.cuh compiled for the CPU)

R, P = bn.R, bn.P
LAM = 0xb3c4d79d41a917585bfc41088d8daaa78b17ea66b99c90dd
KNOBS = ("OG_GLV", "OG_MSM_TAIL", "OG_RED_FAN0")

# ---- mirror of msm.cu's path selection (pick_window, msm_dev, msm_buckets) ------------------------------------------------
RED_FAN_LOG2, TAIL_SLICE, TAIL_THREADS = 3, 512, 128


def pick_window(n):
    return min(max(n.bit_length() - 1 - 3, 2), 16)


def msm_path(curve, n, glv=True, tail=True, fan0=3):
    """Which path a one-shot MSM of n points takes: GLV or not, window bits c, windows W, buckets per window nb, number of
    k_reduce_level launches, and the tail's slice count (0: no tail, the fan-8 levels run to the end)."""
    use_glv = curve == "g1" and glv and n >= 1024
    m = 2 * n if use_glv else n
    c = pick_window(m)
    W = -(-128 // c) if use_glv else -(-255 // c)
    nb = 1 << (c - 1)
    n_in, levels, slices = nb, 0, 0
    while True:
        f = fan0 if levels == 0 else RED_FAN_LOG2
        n_in = (n_in + (1 << f) - 1) >> f
        levels += 1
        if levels == 1 and tail and n_in >= 64 and n_in & (n_in - 1) == 0:
            n_sums, n_slices = n_in.bit_length() + 1, -(-n_in // TAIL_SLICE)
            if n_sums * n_slices <= TAIL_THREADS:
                slices = n_slices
                break
        if n_in <= 1:
            break
    return dict(glv=use_glv, m=m, c=c, W=W, nb=nb, levels=levels, slices=slices)


def heavy_plan(bucket_counts, m, nb):
    """(heavy buckets, heavy segments) of msm_buckets for one-shot MSMs: cap and segment length from the average load m / nb."""
    avg = m // nb
    cap, seg = max(128, 4 * avg), max(2048, 4 * avg)
    heavy = [cnt for cnt in bucket_counts if cnt > cap]
    return len(heavy), sum(-(-cnt // seg) for cnt in heavy), seg


def _n_for(c, glv):
    """An input size whose window is c; odd, so never a multiple of 128 (the last CTA of every per-point kernel is partial)."""
    return (1 << (c + 2 if glv else c + 3)) + 2 * c + 1


# (curve, GLV knob, n): G1 with GLV at c = 8..16, G1 without GLV and G2 at c = 2..16
SWEEP = ([("g1", True, _n_for(c, True)) for c in range(8, 17)] + [("g1", False, _n_for(c, False)) for c in range(2, 17)]
         + [("g2", True, _n_for(c, False)) for c in range(2, 17)])


# ---- digit model (DigitIter::for_each) and the scalar families ------------------------------------------------------------
def signed_digits(s, c, W):
    """[(digit, carry out)] per window of the signed c-bit recoding, and the carry left after the top window."""
    half, out, carry = 1 << (c - 1), [], 0
    for w in range(W):
        v = ((s >> (c * w)) & ((1 << c) - 1)) + carry
        carry = int(v > half)
        out.append((v - (1 << c) if carry else v, carry))
    return out, carry


def _repeat_windows(c, W, raw, bound):
    """sum_{w < J} raw 2^(c w) for the largest J <= W that stays below bound, and J"""
    v, J = 0, 0
    for w in range(W):
        t = v + (raw << (c * w))
        if t >= bound:
            break
        v, J = t, w + 1
    return v, J


def _top_carry(c, W, bound):
    """The largest value below bound whose top window receives a carry: its low c (W - 1) bits exceed the largest value that
    W - 1 digits of at most 2^(c-1) can represent."""
    L = c * (W - 1)
    H = sum((1 << (c - 1)) << (c * i) for i in range(W - 1))
    s = bound - 1
    return s if s & ((1 << L) - 1) > H else ((s >> L) << L) - 1


def edge_values(c, W, bound):
    """{family: [values below bound]} for c-bit windows: digits all +2^(c-1) (top bucket, no negation), all 2^(c-1) + 1
    (negated, carry into every window), all-ones 2^(cj) - 1 (the carry ripples through j windows), bound - 1 / - 2, and the
    largest value whose top window receives a carry."""
    half = 1 << (c - 1)
    top, _ = _repeat_windows(c, W, half, bound)
    neg, _ = _repeat_windows(c, W, half + 1, bound)
    jmax = max(j for j in range(1, W + 1) if (1 << (c * j)) - 1 < bound)
    ones = [(1 << (c * j)) - 1 for j in sorted({1, 2, max(1, jmax // 2), jmax})]
    return dict(top=[top], neg=[neg], ones=ones, below=[bound - 1, bound - 2], top_carry=[_top_carry(c, W, bound)])


# GLV halves are built below this magnitude, inside the region where glv_decompose returns exactly the (k1, k2) a scalar was built
# from: the reduced basis vectors are about 0.87 * 2^127 long and the rounded coefficients may be off by 1/8 of a unit, so pairs of
# magnitude up to (1/2 - 1/8) * 0.87 * 2^127 come back unchanged.  Uniform scalars reach the decomposition's larger outputs.
GLV_BOUND = int(0.32 * 2**127)


def glv_edge_pairs(c):
    """[(k, (|k1|, neg1), (|k2|, neg2))]: digit patterns of edge_values on the 127-bit halves, with every sign combination,
    folded into k = k1 + k2 lambda mod r."""
    W = -(-128 // c)
    vals = [v for vs in edge_values(c, W, GLV_BOUND).values() for v in vs]
    out = []
    for i, a in enumerate(vals):
        b = vals[(i * 3 + 1) % len(vals)]
        for n1, n2 in ((0, 0), (0, 1), (1, 0), (1, 1)):
            out.append((((-a if n1 else a) + (-b if n2 else b) * LAM) % R, (a, n1), (b, n2)))
    return out


def scalar_sets(curve, n, glv, rng):
    """Two scalar lists for one case: a mix of uniform scalars in [0, r) and every edge family built for this case's c, and a
    mostly-zero list that leaves most buckets empty."""
    p = msm_path(curve, n, glv)
    if p["glv"]:
        edges = [k for k, _, _ in glv_edge_pairs(p["c"])] + [R - 1, R - 2]
    else:
        edges = [v for vs in edge_values(p["c"], p["W"], R).values() for v in vs]
    mixed = [rng.randrange(R) if i % 3 else edges[(i // 3) % len(edges)] for i in range(n)]
    mixed[:len(edges)] = edges                                        # every edge value at least once, also at n = 37
    sparse = [0] * n
    for i in rng.sample(range(n), max(1, n // 40)):
        sparse[i] = rng.choice([rng.randrange(R), rng.choice(edges)])
    return mixed, sparse


# ---- CPU tests: the table covers every path, and the scalar families are what they claim ------------------------------------
def test_sweep_table_covers_every_msm_path():
    rows = {(curve, glv): {} for curve, glv, _ in SWEEP}
    for curve, glv, n in SWEEP:
        p = msm_path(curve, n, glv)
        assert p["glv"] == (curve == "g1" and glv), (curve, glv, n)
        assert n % 128 != 0 and p["m"] % 128 != 0, (curve, n)
        rows[(curve, glv)][p["c"]] = p
    assert sorted(rows[("g1", True)]) == list(range(8, 17))
    assert sorted(rows[("g1", False)]) == list(range(2, 17))
    assert sorted(rows[("g2", True)]) == list(range(2, 17))
    for curve in ("g1", "g2"):
        slices = {p["slices"] for (cv, _), ps in rows.items() if cv == curve for p in ps.values()}
        assert {0, 1, 2, 4, 8} <= slices, curve
    # fixed points of the mirror: the tail starts where nb >> fan0 reaches 64, its slices double from c = 14
    assert [msm_path("g2", _n_for(c, False))["slices"] for c in range(8, 17)] == [0, 0, 1, 1, 1, 1, 2, 4, 8]
    assert [msm_path("g2", _n_for(c, False), fan0=5)["slices"] for c in range(10, 17)] == [0, 0, 1, 1, 1, 1, 2]
    assert msm_path("g2", _n_for(12, False), tail=False)["levels"] == 4           # 2048 -> 256 -> 32 -> 4 -> 1
    assert msm_path("g2", _n_for(12, False), tail=False, fan0=5)["levels"] == 3   # 2048 -> 64 -> 8 -> 1
    p = msm_path("g1", 1 << 20)
    assert (p["glv"], p["c"], p["W"], p["slices"], p["levels"]) == (True, 16, 8, 8, 1)
    assert msm_path("g1", 1023)["glv"] is False and msm_path("g1", 1024)["glv"] is True
    assert msm_path("g1", 1 << 20, glv=False)["W"] == 16


def test_scalar_families_hit_their_digits():
    """Every edge family does to the signed-digit recoding what its name says, for every c and both scalar lengths."""
    for c in range(2, 17):
        for W, bound in ((-(-255 // c), R), (-(-128 // c), GLV_BOUND))[:2 if c >= 8 else 1]:      # GLV runs at c >= 8
            e = edge_values(c, W, bound)
            half = 1 << (c - 1)
            for fam, vals in e.items():
                for v in vals:
                    assert 0 <= v < bound, (c, fam)
                    _, last = signed_digits(v, c, W)
                    assert last == 0, (c, fam)                             # the top window absorbs the last carry
            d, _ = signed_digits(e["top"][0], c, W)
            J = next(w for w in range(W + 1) if w == W or d[w][0] == 0)
            assert J >= 2 and all(x == (half, 0) for x in d[:J]), c        # top bucket nb - 1, never negated
            d, _ = signed_digits(e["neg"][0], c, W)
            J = next(w for w in range(W) if d[w][1] == 0)
            assert J >= 2 and all(cy == 1 and x <= 0 for x, cy in d[:J]), c   # negated, carry into every window up to J
            for v in e["ones"]:
                j = v.bit_length() // c
                d, _ = signed_digits(v, c, W)
                assert [x for x, _ in d[:j]] == [-1] + [0] * (j - 1) and d[j][0] == 1, (c, j)   # ripple into window j
            d, _ = signed_digits(e["top_carry"][0], c, W)
            assert d[W - 2][1] == 1, c                                     # the top window receives a carry


def test_glv_edge_pairs_decompose_as_built(h):      # noqa: F811
    """glv_decompose (glv.cuh, host build) returns exactly the halves and signs every GLV edge scalar was built from, so the GLV
    rows of the sweep put their digit patterns where they claim to."""
    import ctypes as C
    pairs = [x for c in range(8, 17) for x in glv_edge_pairs(c)]
    out = C.create_string_buffer(65 * len(pairs))
    h.ht_glv_decompose(b"".join(k.to_bytes(32, "little") for k, _, _ in pairs), out, C.c_uint64(len(pairs)))
    for i, (k, (a, n1), (b, n2)) in enumerate(pairs):
        rec = out.raw[65 * i:65 * i + 65]
        m1, m2, sg = int.from_bytes(rec[:32], "little"), int.from_bytes(rec[32:64], "little"), rec[64]
        assert (m1, m2) == (a, b), hex(k)
        assert (bool(sg & 1), bool(sg & 2)) == (bool(n1 and a), bool(n2 and b)), hex(k)
    assert max(max(a, b) for _, (a, _), (b, _) in pairs) > 0.3 * 2**127


# ---- GPU helpers ---------------------------------------------------------------------------------------------------------
GEN = {"g1": bn.g1_to_bytes(bn.G1_GEN), "g2": bn.g2_to_bytes(bn.G2_GEN)}
PB = {"g1": 64, "g2": 128}
DIRECT_ORACLE_MAX = 1 << 13            # up to here the oracle's CPU MSM is run on the same bytes as well


def _neg(curve, pt):
    if curve == "g1":
        return pt[:32] + ((P - int.from_bytes(pt[32:], "little")) % P).to_bytes(32, "little")
    y0, y1 = int.from_bytes(pt[64:96], "little"), int.from_bytes(pt[96:], "little")
    return pt[:64] + ((P - y0) % P).to_bytes(32, "little") + ((P - y1) % P).to_bytes(32, "little")


def make_points(ctx, curve, n, rng, exceptional=True):
    """n points d_i G with their discrete logs d_i; with `exceptional`, also points at infinity, duplicates and P / -P pairs."""
    d = [rng.randrange(1, R) for _ in range(n)]
    gen = ctx.g1_generator_mul if curve == "g1" else ctx.g2_generator_mul
    pts = bytearray(gen(cport.frs(d)))
    pb = PB[curve]
    k = min(16, n)
    fixed = cport.g1_fixed_mul_batch if curve == "g1" else cport.g2_fixed_mul_batch
    assert bytes(pts[:pb * k]) == fixed(GEN[curve], cport.frs(d[:k]))
    if exceptional and n >= 8:
        for i in rng.sample(range(n), max(1, n // 500)):              # infinity
            pts[pb * i:pb * i + pb] = bytes(pb); d[i] = 0
        for _ in range(max(1, n // 500)):                              # duplicates
            i, j = rng.randrange(n), rng.randrange(n)
            pts[pb * i:pb * i + pb] = pts[pb * j:pb * j + pb]; d[i] = d[j]
        for _ in range(max(1, n // 500)):                              # P, -P
            i, j = rng.randrange(n), rng.randrange(n)
            pts[pb * i:pb * i + pb] = _neg(curve, bytes(pts[pb * j:pb * j + pb])); d[i] = (R - d[j]) % R
    return bytes(pts), d


def expected(curve, d, ks, pts=None):
    """sum k_i (d_i G) by the oracle: one fixed-base multiplication, and the CPU MSM on the same bytes when it is cheap."""
    t = sum(a * b for a, b in zip(d, ks)) % R
    fixed = cport.g1_fixed_mul_batch if curve == "g1" else cport.g2_fixed_mul_batch
    exp = fixed(GEN[curve], cport.frs([t]))
    if pts is not None and len(d) <= DIRECT_ORACLE_MAX:
        msm = cport.g1_msm if curve == "g1" else cport.g2_msm
        assert msm(pts, cport.frs(ks)) == exp
    return exp


def run_profiled(ctx, curve, pts, sc):
    """One MSM with the per-kernel profile on -> (result bytes, {kernel: launches})."""
    ctx.profile(True)
    try:
        ctx.profile_dump()
        out = (ctx.msm_g1 if curve == "g1" else ctx.msm_g2)(pts, sc)
        prof = ctx.profile_dump()
    finally:
        ctx.profile(False)
    return out, {k: v[0] for k, v in prof.items()}


def check_path(prof, curve, p):
    """The kernels that ran are the ones the mirror predicts."""
    g = "g1" if curve == "g1" else "g2"
    assert prof.get("k_glv_expand", 0) == (1 if p["glv"] else 0), prof
    assert prof.get(f"k_tail_sums_{g}", 0) == (1 if p["slices"] else 0), (p, prof)
    assert prof.get(f"k_tail_finish_{g}", 0) == (1 if p["slices"] else 0), (p, prof)
    assert prof.get(f"k_reduce_level_{g}", 0) == p["levels"], (p, prof)


@pytest.fixture
def knobs(monkeypatch):
    """Each test starts from the default knobs and sets its own."""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


# ---- one-shot window sweep --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("curve,glv,n", SWEEP, ids=[f"{cv}-{'glv' if g and cv == 'g1' else 'plain'}-c{msm_path(cv, n, g)['c']}"
                                                     for cv, g, n in SWEEP])
def test_msm_window_sweep_vs_oracle(ctx, knobs, curve, glv, n):
    knobs.setenv("OG_GLV", "1" if glv else "0")
    rng = random.Random(1000 * n + (curve == "g2") * 7 + glv)
    p = msm_path(curve, n, glv)
    pts, d = make_points(ctx, curve, n, rng)
    for ks in scalar_sets(curve, n, glv, rng):
        sc = cport.frs(ks)
        got, prof = run_profiled(ctx, curve, pts, sc)
        assert got == expected(curve, d, ks, pts), (curve, glv, n, p)
        check_path(prof, curve, p)


# ---- heavy buckets ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["g1", "g2"])
def test_msm_heavy_buckets_beyond_one_grid(ctx, knobs, curve):
    """2^20 points whose scalars are small (only window 0 has digits): half of them in one bucket (256 segments: the 32-lane loop
    of k_heavy_combine goes round 8 times, for G2 too), the rest spread over SM count + 8 further buckets.  More heavy segments
    than k_bucket_heavy's 4 x SM-count CTAs (its grid-stride loop runs twice) and more heavy buckets than k_heavy_combine's
    SM-count CTAs."""
    import torch
    sm = torch.cuda.get_device_properties(ctx.device).multi_processor_count
    rng = random.Random(4242 if curve == "g1" else 4243)
    n = 1 << 20
    K = sm + 8
    ks = [1 if i % 2 == 0 else 2 + (i // 2) % K for i in range(n)]
    p = msm_path(curve, n)
    counts = [n // 2] + [(n // 2) // K + (v < (n // 2) % K) for v in range(K)]
    n_heavy, n_seg, seg = heavy_plan(counts, p["m"], p["nb"])
    assert n_heavy == K + 1 > sm and n_seg > 4 * sm and n // 2 > 32 * seg, (n_heavy, n_seg, sm)
    pts, d = make_points(ctx, curve, n, rng, exceptional=False)
    got, prof = run_profiled(ctx, curve, pts, cport.frs(ks))
    assert got == expected(curve, d, ks)
    assert prof.get(f"k_bucket_heavy_{curve}") == 1


# ---- knob matrix ------------------------------------------------------------------------------------------------------------
# G1 and G2 cases on both sides of the tail threshold (c >= 7 + fan0) for every fan0: G1 2^11 + 19 points are c = 9 with GLV and
# c = 8 without, 2^15 + 19 are c = 13 / 12; G2 2^12 + 19 and 2^16 + 19 points are c = 9 and 13
KNOB_CASES = [("g1", (1 << 11) + 19), ("g1", (1 << 15) + 19), ("g2", (1 << 12) + 19), ("g2", (1 << 16) + 19)]


@pytest.fixture(scope="module")
def knob_inputs(ctx):
    rng = random.Random(99)
    out = []
    for curve, n in KNOB_CASES:
        pts, d = make_points(ctx, curve, n, rng)
        ks = [rng.randrange(R) for _ in range(n)]
        for i, v in enumerate([0, 1, R - 1, R - 2, 2**127 - 1, 2**128, LAM, R - LAM]):
            ks[3 * i] = v
        out.append((curve, n, pts, cport.frs(ks), expected(curve, d, ks, pts)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fan0", [3, 4, 5])
@pytest.mark.parametrize("tail", [0, 1])
@pytest.mark.parametrize("glv", [0, 1])
def test_msm_knob_matrix(ctx, knobs, knob_inputs, glv, tail, fan0):
    knobs.setenv("OG_GLV", str(glv)); knobs.setenv("OG_MSM_TAIL", str(tail)); knobs.setenv("OG_RED_FAN0", str(fan0))
    tails = set()
    for curve, n, pts, sc, exp in knob_inputs:
        p = msm_path(curve, n, glv=bool(glv), tail=bool(tail), fan0=fan0)
        got, prof = run_profiled(ctx, curve, pts, sc)
        assert got == exp, (curve, n, p)
        check_path(prof, curve, p)
        tails.add(bool(p["slices"]))
    assert tails == ({False, True} if tail else {False})


@pytest.mark.gpu
def test_msm_knobs_read_on_every_call(ctx, knobs, knob_inputs):
    """Each knob set AFTER an MSM has run in this process takes effect on the next call (the knobs used to be frozen at the first
    MSM of the process, so a test toggling them checked the default path twice)."""
    curve, n, pts, sc, exp = knob_inputs[1]                     # G1, c = 13 with GLV: the tail runs by default
    got, prof = run_profiled(ctx, curve, pts, sc)
    assert got == exp
    check_path(prof, curve, msm_path(curve, n))
    for env, kw in (("OG_GLV", dict(glv=False)), ("OG_MSM_TAIL", dict(glv=False, tail=False)),
                    ("OG_RED_FAN0", dict(glv=False, tail=False, fan0=5))):
        knobs.setenv(env, {"OG_GLV": "0", "OG_MSM_TAIL": "0", "OG_RED_FAN0": "5"}[env])
        got, prof = run_profiled(ctx, curve, pts, sc)
        assert got == exp, env
        check_path(prof, curve, msm_path(curve, n, **kw))
    for env in KNOBS:
        knobs.delenv(env)
    got, prof = run_profiled(ctx, curve, pts, sc)
    assert got == exp
    check_path(prof, curve, msm_path(curve, n))


# ---- prover at non-default window bits -------------------------------------------------------------------------------------
PROVER_KNOBS = ("OG_C_A", "OG_C_B", "OG_C_C", "OG_WINDOW_BITS", "OG_RED_FAN0", "OG_LANE_PRIO", "OG_GLV", "OG_MSM_TAIL")
PROVER_SETTINGS = [
    # every row of DESIGN.md section 8's window sweep
    ("16-15-16", dict(OG_C_A="16", OG_C_B="15", OG_C_C="16")),
    ("15-15-15", dict(OG_C_A="15", OG_C_B="15", OG_C_C="15")),
    ("16-16-16", dict(OG_C_A="16", OG_C_B="16", OG_C_C="16")),
    ("14-14-15", dict(OG_C_A="14", OG_C_B="14", OG_C_C="15")),
    ("14-14-14", dict(OG_C_A="14", OG_C_B="14", OG_C_C="14")),
    ("8-9-10", dict(OG_C_A="8", OG_C_B="9", OG_C_C="10")),              # many windows, long bucket lists
    ("window-bits-13", dict(OG_WINDOW_BITS="13")),
    ("window-bits-0", dict(OG_WINDOW_BITS="0")),                          # out of range or not a number: the defaults
    ("window-bits-1", dict(OG_WINDOW_BITS="1")),
    ("window-bits-17", dict(OG_WINDOW_BITS="17")),
    ("window-bits-abc", dict(OG_WINDOW_BITS="abc", OG_C_C="17")),
    ("red-fan0-4", dict(OG_RED_FAN0="4")),
    ("red-fan0-5", dict(OG_RED_FAN0="5")),
    ("lane-prio-0", dict(OG_LANE_PRIO="0")),                              # in a context created after setting it
]
PROVER_BATCH = 6


@pytest.fixture(scope="module")
def keys32(ctx):
    return withdraw_keys32(ctx)


@pytest.fixture(scope="module")
def prover_default(ctx, keys32):
    """The seeded batch proved at the default settings in two chunks; proof 0 against the oracle's C prover."""
    pk, vk, cs, pkb, vkb = keys32
    rng = random.Random(616)
    inputs = rand_inputs(rng, PROVER_BATCH, 32)
    rs = cport.frs([rng.randrange(R) for _ in range(2 * PROVER_BATCH)])
    saved = {k: os.environ.pop(k) for k in PROVER_KNOBS + ("OG_CHUNK", "OG_LANES") if k in os.environ}
    os.environ["OG_CHUNK"] = "4"
    try:
        PK = ob.ProvingKey(ctx, pk)
        proofs, pub = ob.prove(PK, *inputs, rs)
        PK.close()
    finally:
        os.environ.pop("OG_CHUNK")
        os.environ.update(saved)
    nul, sec, rec, sib, bits = inputs
    wit = cport.withdraw_witness(nul[:32], sec[:32], rec[:32], sib[:32 * 32], bits[:1], 32)
    assert proofs[:256] == cport.Prover(cs, pkb).prove_batch(wit, rs[:64])
    return inputs, rs, proofs, pub


@pytest.mark.gpu
@pytest.mark.parametrize("env", [e for _, e in PROVER_SETTINGS], ids=[i for i, _ in PROVER_SETTINGS])
def test_prover_window_bits_and_knobs_reproduce_default(ctx, keys32, prover_default, monkeypatch, env):
    """Proofs are deterministic in (pk, witness, r, s): every window setting and knob must give the default setting's bytes (and the
    default is pinned to the oracle's C prover), over a batch of two chunks proved on two lanes."""
    pk, vk = keys32[0], keys32[1]
    inputs, rs, ref, ref_pub = prover_default
    for k in PROVER_KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("OG_CHUNK", "4"); monkeypatch.setenv("OG_LANES", "2")
    c = ob.Context(ctx.device) if "OG_LANE_PRIO" in env else ctx
    try:
        PK = ob.ProvingKey(c, pk)                  # window bits are read when the key is loaded
        try:
            proofs, pub = ob.prove(PK, *inputs, rs)
        finally:
            PK.close()
    finally:
        if c is not ctx:
            c.close()
    assert pub == ref_pub
    for i in range(PROVER_BATCH):
        assert proofs[256 * i:256 * i + 256] == ref[256 * i:256 * i + 256], i
    assert ob.verify(vk, pub[-96:], proofs[-256:])
