"""The bucket stage of the MSM engine (msm.cu: msm_buckets) on crafted bucket lists, against known discrete logs.

Scalars decide which bucket a point goes to, not what the bucket's running sum is when the next point arrives, so through
og_msm_g1/g2 and the prover the exceptional branches of the group law are reached only where a collision is trivial (an
accumulator still holding the first point of its run).  og_msm_bucket_sums runs the real msm_buckets of the G1 or G2 unit on bucket
lists the test chooses, so the collisions are placed on purpose:

  * accumulation (k_bucket_acc_sm1 / k_bucket_acc_sm): acc == q and acc == -q with a general Z (zz != 1), restarts after infinity,
    negated infinity entries, a list of exactly `cap` entries;
  * heavy buckets (k_heavy_plan, k_bucket_heavy, k_heavy_combine): lists at the cap and at the segment length, segment sums that
    cancel, are equal, or are infinity, trees whose every level doubles, more heavy buckets than one scan round of k_heavy_plan;
  * reduction (k_reduce_level(_sm), k_group_total): R + S = infinity / 2R, T + R = 2R / infinity, U + S = infinity / 2S, at
    OG_RED_FAN0 = 3, 4 and 5;
  * the one-shot tail (k_tail_sums / k_tail_finish) with colliding Q_k sums, and the prover's shape (64 groups of 2^14 / 2^15
    buckets, mostly empty).

Every table point is d_i G, so every bucket and every group total is (sum of +-weight d_i mod r) G: one fixed-base multiplication by
the oracle's C port, exact at any size.  `simulate` below restates the kernels' order of operations over the logs mod r and counts
the exceptional events of each kernel; a CPU test asserts that every case reaches the branches it is named after (for the G1 and G2
thread counts of k_bucket_heavy), so the case table stays honest when the kernels' order changes.  The GPU tests compare the probe's
totals and buckets with the oracle byte for byte and check the per-kernel profile against the simulator."""
import ctypes as C
import random

import pytest

from owshen_b200 import api
from oracle import bn254 as bn
from oracle import cport

R = bn.R
HEAVY_THREADS = {"g1": 256, "g2": 128}          # k_bucket_heavy<F, HT>
COMBINE_LANES, RED_FAN_LOG2, TAIL_SLICE, TAIL_THREADS = 32, 3, 512, 128
EVENTS = ("acc_dbl", "acc_cancel",              # k_bucket_acc: acc == q / acc == -q with zz != 1
          "seg_inf", "heavy_dbl", "heavy_cancel",   # k_bucket_heavy: a segment sums to infinity; equal / opposite operands
          "combine_dbl", "combine_cancel",      # k_heavy_combine: equal / opposite segment sums
          "rs_inf", "rs_dbl", "tr_dbl", "tr_inf",   # k_reduce_level: R + S = inf / 2R, T + R = 2R / inf
          "tot_inf", "tot_dbl",                 # k_group_total: U + S = inf / 2S
          "tail_dbl", "tail_inf")               # k_tail_sums / k_tail_finish: equal / opposite operands
GEN = {"g1": bn.g1_to_bytes(bn.G1_GEN), "g2": bn.g2_to_bytes(bn.G2_GEN)}
PB = {"g1": 64, "g2": 128}


# ---- integer model of msm_buckets over the discrete logs (None = the point at infinity) --------------------------------------
def _add(ev, a, b, dbl, inf):
    """a + b, counting the exceptional branch of the group law (both finite and equal, or opposite)"""
    if b is None:
        return a
    if a is None:
        return b
    if a == b:
        ev[dbl] += 1
        return 2 * a % R
    s = (a + b) % R
    if s == 0:
        ev[inf] += 1
        return None
    return s


def _mul2(a, k):
    return None if a is None else a * pow(2, k, R) % R


def _thread_bucket(ev, vals):
    """k_bucket_acc_sm1 / k_bucket_acc_sm: one thread, list order; `fresh` = the accumulator holds one point (zz = 1)"""
    acc, fresh = None, False
    for v in vals:
        if v is None:
            continue
        if acc is None:
            acc, fresh = v, True
            continue
        if not fresh and acc == v:
            ev["acc_dbl"] += 1
        if not fresh and (acc + v) % R == 0:
            ev["acc_cancel"] += 1
        acc = _add(ev, acc, v, "_", "_")
        fresh = False
    return acc


def _tree(ev, a, n, dbl, inf):
    s = n // 2
    while s:
        for t in range(s):
            a[t] = _add(ev, a[t], a[t + s], dbl, inf)
        s //= 2
    return a[0]


def _heavy_bucket(ev, vals, seg, ht):
    """k_bucket_heavy: one CTA per segment of `seg` entries, thread t takes entries t, t + ht, ..., then a shared-memory tree;
    k_heavy_combine: lane l adds segment sums l, l + 32, ..., then a warp tree"""
    partials = []
    for k0 in range(0, len(vals), seg):
        s = vals[k0:k0 + seg]
        sh = [None] * ht
        for t in range(ht):
            for v in s[t::ht]:
                sh[t] = _add(ev, sh[t], v, "heavy_dbl", "heavy_cancel")
        p = _tree(ev, sh, ht, "heavy_dbl", "heavy_cancel")
        if p is None:
            ev["seg_inf"] += 1
        partials.append(p)
    lanes = [None] * COMBINE_LANES
    for lane in range(COMBINE_LANES):
        for p in partials[lane::COMBINE_LANES]:
            lanes[lane] = _add(ev, lanes[lane], p, "combine_dbl", "combine_cancel")
    return _tree(ev, lanes, COMBINE_LANES, "combine_dbl", "combine_cancel")


def _level(ev, S, U, n_in, f, w):
    """k_reduce_level(_sm) for one group: parent p runs R, T over its children from the top down"""
    n_out = (n_in + (1 << f) - 1) >> f
    So, Uo = [None] * n_out, [None] * n_out
    for p in range(n_out):
        lo, hi = p << f, min(n_in, (p << f) + (1 << f))
        if not any(x is not None for x in S[lo:hi]) and (U is None or not any(x is not None for x in U[lo:hi])):
            continue
        Rr = T = None
        for i in range(hi - 1, lo, -1):
            Rr = _add(ev, Rr, S[i], "rs_dbl", "rs_inf")
            T = _add(ev, T, Rr, "tr_dbl", "tr_inf")
        Rr = _add(ev, Rr, S[lo], "rs_dbl", "rs_inf")
        T = _mul2(T, w)
        if U is not None:
            for i in range(lo, hi):
                T = _add(ev, T, U[i], "_", "_")
        So[p], Uo[p] = Rr, T
    return So, Uo


def _tail(ev, Rs, Ts, n1, f):
    """k_tail_sums (sum T, sum R and Q_k = the R_p whose index has bit k set; strided additions, then a tree) and k_tail_finish"""
    n_bits = n1.bit_length() - 1
    n_sums, n_slices = n_bits + 2, -(-n1 // TAIL_SLICE)
    part = []
    for q in range(n_sums):
        for sl in range(n_slices):
            a = [None] * TAIL_THREADS
            for tid in range(TAIL_THREADS):
                if q < 2:
                    src = Ts if q == 0 else Rs
                    idx = range(sl * TAIL_SLICE + tid, min(n1, sl * TAIL_SLICE + TAIL_SLICE), TAIL_THREADS)
                else:
                    k = q - 2
                    js = range(sl * (TAIL_SLICE // 2) + tid, min(n1 >> 1, sl * (TAIL_SLICE // 2) + TAIL_SLICE // 2), TAIL_THREADS)
                    src, idx = Rs, [((j >> k) << (k + 1)) | (1 << k) | (j & ((1 << k) - 1)) for j in js]
                for p in idx:
                    a[tid] = _add(ev, a[tid], src[p], "tail_dbl", "tail_inf")
            part.append(_tree(ev, a, TAIL_THREADS, "tail_dbl", "tail_inf"))
    s = n_slices // 2
    while s:
        for t in range(n_sums * n_slices):
            if t % n_slices < s:
                part[t] = _add(ev, part[t], part[t + s], "tail_dbl", "tail_inf")
        s //= 2
    v = None
    for k in range(n_sums - 3, -1, -1):
        v = _add(ev, _mul2(v, 1), part[(2 + k) * n_slices], "tail_dbl", "tail_inf")
    v = _add(ev, _mul2(v, f), part[0], "tail_dbl", "tail_inf")
    return _add(ev, v, part[n_slices], "tail_dbl", "tail_inf")


def plan(case):
    """cap and segment length of msm_buckets (test_msm_paths.heavy_plan restates them for one-shot MSMs)"""
    avg = case.n_entries_max // case.n_keys
    return max(128, 4 * avg), max(2048, 4 * avg)


def simulate(case, curve):
    """-> dict(totals, buckets, events, levels (k_reduce_level launches), tail (k_tail_* ran), heavy (buckets over the cap))"""
    ev = dict.fromkeys(EVENTS + ("_",), 0)
    cap, seg = plan(case)
    B = [None] * case.n_keys
    heavy = 0
    for key, lst in case.lists.items():
        vals = [case.val(e) for e in lst]
        if len(vals) > cap:
            heavy += 1
            B[key] = _heavy_bucket(ev, vals, seg, HEAVY_THREADS[curve])
        else:
            B[key] = _thread_bucket(ev, vals)
    fan0 = case.fan0 or RED_FAN_LOG2
    totals, levels, tail = [], 0, False
    for g in range(case.n_groups):
        S, U, n_in, w, lv = B[g * case.nb:(g + 1) * case.nb], None, case.nb, 0, 0
        while True:
            f = fan0 if U is None else RED_FAN_LOG2
            S, U = _level(ev, S, U, n_in, f, w)
            n_in, w, lv = len(S), w + f, lv + 1
            if case.few_groups and lv == 1 and case.tail and n_in >= 64 and n_in & (n_in - 1) == 0:
                n_sums, n_slices = n_in.bit_length() + 1, -(-n_in // TAIL_SLICE)
                if n_sums * n_slices <= TAIL_THREADS:
                    totals.append(_tail(ev, S, U, n_in, w))
                    tail = True
                    break
            if n_in <= 1:
                totals.append(_add(ev, U[0], S[0], "tot_dbl", "tot_inf"))
                break
        levels = lv
    del ev["_"]
    return dict(totals=totals, buckets=B, events=ev, levels=levels, tail=tail, heavy=heavy)


# ---- the cases --------------------------------------------------------------------------------------------------------------
class Case:
    """Bucket lists over a table of points with known logs; point 0 is the point at infinity.  An entry is (index << 1) | negate."""

    def __init__(self, name, n_groups, nb, seed, expect, fan0=None, few_groups=False, tail=True, n_entries_max=None,
                 buckets=True):
        self.name, self.n_groups, self.nb, self.n_keys = name, n_groups, nb, n_groups * nb
        self.rng = random.Random(seed)
        self.expect, self.fan0, self.few_groups, self.tail, self.buckets = set(expect), fan0, few_groups, tail, buckets
        self._nmax = n_entries_max
        self.logs = [0]
        self.lists = {}

    INF, NEG_INF = 0, 1

    def pt(self, d):
        """entry of a new table point with log d"""
        self.logs.append(d % R)
        return (len(self.logs) - 1) << 1

    def rnd(self):
        return self.pt(self.rng.randrange(1, R))

    def val(self, e):
        d = self.logs[e >> 1] * (-1 if e & 1 else 1) % R
        return d or None

    def put(self, key, *entries):
        assert 0 <= key < self.n_keys and key not in self.lists
        self.lists[key] = list(entries)

    def fill(self, n_buckets, max_len=6, groups=None):
        """random lists of random points in empty buckets (of the given groups)"""
        gs = range(self.n_groups) if groups is None else groups
        for _ in range(n_buckets):
            key = self.rng.choice(gs) * self.nb + self.rng.randrange(self.nb)
            if key not in self.lists:
                self.put(key, *[self.rnd() ^ self.rng.randrange(2) for _ in range(self.rng.randrange(1, max_len + 1))])

    @property
    def counts(self):
        c = [0] * self.n_keys
        for k, lst in self.lists.items():
            c[k] = len(lst)
        return c

    @property
    def entries(self):
        return [e for k in sorted(self.lists) for e in self.lists[k]]

    @property
    def n_entries_max(self):
        return self._nmax if self._nmax is not None else sum(len(v) for v in self.lists.values())


def case_acc_deep():
    """Accumulation below the cap: deep doubling and cancellation with a general Z, restarts, several cancellations in one list,
    negated infinity entries; 3 x 64 keys (not a multiple of 128)."""
    c = Case("acc-deep", 3, 64, 1, {"acc_dbl", "acc_cancel"})
    for g in range(3):
        k = g * 64
        a, b = c.rnd(), c.rnd()
        ab = c.val(a) + c.val(b)
        c.put(k + 0, a, b, c.pt(ab))                                     # P1 + P2 meets (d1 + d2) G: doubling, zz != 1
        c.put(k + 5, a, b, c.pt(-ab), c.rnd(), c.rnd())                   # cancels deep, then restarts
        lst = []
        for _ in range(4):                                                # several cancellations in one list
            x, y = c.rnd(), c.rnd()
            lst += [x, y, c.pt(-(c.val(x) + c.val(y)))]
        c.put(k + 7, *lst, c.rnd())
        c.put(k + 9, c.NEG_INF, a, c.NEG_INF, b ^ 1, c.INF, c.pt(-(c.val(a) - c.val(b))), c.NEG_INF, c.rnd())
        c.put(k + 63, a, b, c.pt(ab), c.pt(-2 * ab), c.rnd(), c.rnd())   # doubling, then the double cancels, restart
        c.put(k + 33, c.NEG_INF, c.INF)                                   # only infinities
    c.fill(60)
    return c


def case_cap_boundary():
    """A point repeated exactly `cap` times stays on the thread path; cap + 1 copies go to k_bucket_heavy, whose thread partials
    are then equal; 512 entries +-Q by parity (the same for 256 and 128 threads) double at every tree level and cancel at the
    top; 512 copies of Q double at every level.  n_entries_max = 2048 over 64 keys: cap 128."""
    c = Case("cap-boundary", 1, 64, 2, {"heavy_dbl", "heavy_cancel", "seg_inf"}, n_entries_max=2048)
    p, q = c.rnd(), c.rnd()
    c.put(0, *[p] * 128)
    c.put(1, *[p] * 129)
    c.put(2, *[q ^ (k & 1) for k in range(512)])
    c.put(3, *[q] * 512)
    c.fill(20)
    return c


def case_segments():
    """Lists of seg - 1, seg, seg + 1 and 2 seg entries; two segments that cancel, two equal ones, and an infinite segment between
    two finite ones (cap 128, seg 2048)."""
    c = Case("segments", 1, 4096, 3, {"combine_cancel", "combine_dbl", "seg_inf", "heavy_cancel"}, buckets=True)
    pool = [c.rnd() for _ in range(512)]
    rl = lambda n: [c.rng.choice(pool) ^ c.rng.randrange(2) for _ in range(n)]
    for key, n in enumerate((2047, 2048, 2049, 4096)):
        c.put(key, *rl(n))
    L = rl(2048)
    c.put(4, *L, *[e ^ 1 for e in L])                                     # segment sums X and -X: the combine cancels
    c.put(5, *L, *L)                                                      # equal segment sums: the combine doubles
    M = rl(1024)
    c.put(6, *rl(2048), *M, *[e ^ 1 for e in M], *rl(100))               # the middle segment sums to infinity
    c.fill(40)
    return c


def case_many_heavy():
    """300 heavy buckets over 4 groups (k_heavy_plan scans them in two rounds of 256): half of them cancel to infinity, half
    are one half-list twice."""
    c = Case("many-heavy", 4, 1024, 4, {"seg_inf", "heavy_cancel"}, buckets=True)
    keys = c.rng.sample(range(c.n_keys), 300)
    for i, key in enumerate(keys):
        M = [c.rnd() ^ c.rng.randrange(2) for _ in range(65)]
        c.put(key, *M, *([e ^ 1 for e in M] if i % 2 else M))
    c.fill(100)
    return c


def _plant_reduction(c, g, f, chunk0=0):
    """in group g, fan-0 width 2^f: chunks whose running sums R cancel and restart, R doubles, T + R doubles, T + R cancels"""
    F = 1 << f
    top = lambda j: g * c.nb + (chunk0 + j) * F + F - 1
    x = c.rnd()
    c.put(top(0), x); c.put(top(0) - 1, x ^ 1); c.put(top(0) - 2, c.rnd())     # R = X, R - X = inf, restart
    y = c.rnd()
    c.put(top(1), y); c.put(top(1) - 1, y)                                     # R + X = 2R
    z = c.rnd()
    c.put(top(2), z); c.put(top(2) - 2, c.rnd())                               # empty child: T + R = 2R
    a = c.rnd()
    c.put(top(3), a); c.put(top(3) - 1, c.pt(-2 * c.val(a)))                   # R = -a after T = a: T + R = inf
    for j in range(4):
        c.put(top(j) - F + 1, c.rnd())                                          # the chunk's first bucket


def case_reduction(fan0):
    c = Case(f"reduction-fan{fan0}", 2, 256, 10 + fan0, {"rs_inf", "rs_dbl", "tr_dbl", "tr_inf"}, fan0=fan0)
    for g in range(2):
        _plant_reduction(c, g, fan0)
    return c


def case_group_totals():
    """nb = 8: one level, then k_group_total: only bucket 1 filled (U = S: doubles), B0 = 2X and B1 = -X (U = -S: cancels),
    all buckets equal"""
    c = Case("group-totals", 3, 8, 20, {"tot_dbl", "tot_inf", "rs_dbl"})
    c.put(1, c.rnd())
    x = c.rnd()
    c.put(8, c.pt(2 * c.val(x))); c.put(9, x ^ 1)
    z = c.rnd()
    for b in range(8):
        c.put(16 + b, z)
    return c


def case_tail(tail):
    """few_groups with nb = 512: R_p = the chunk sums are all X (group 0) or +-X by the parity of p (group 1), so the Q_k trees
    double and cancel; with the tail off the fan-8 levels meet the same collisions"""
    c = Case("tail" if tail else "tail-off", 2, 512, 30, {"tail_dbl", "tail_inf"} if tail else {"rs_dbl", "rs_inf"},
             few_groups=True, tail=tail)
    x, y = c.rnd(), c.rnd()
    for p in range(64):
        c.put(8 * p, x)
        c.put(512 + 8 * p, y ^ (p & 1))
    c.put(3, c.rnd()); c.put(512 + 77, c.rnd())
    return c


def case_prover(log_nb):
    """the prover's shape: 64 groups of 2^14 or 2^15 buckets, mostly empty; reduction and accumulation collisions planted in a
    few groups, one heavy bucket"""
    c = Case(f"prover-2^{log_nb}", 64, 1 << log_nb, 40 + log_nb,
             {"rs_inf", "rs_dbl", "tr_dbl", "tr_inf", "acc_dbl", "acc_cancel", "heavy_cancel", "tot_dbl"}, buckets=False)
    for g in (3, 31, 63):
        _plant_reduction(c, g, RED_FAN_LOG2, chunk0=(1 << (log_nb - 3)) - 4)   # the top four chunks
        a, b = c.rnd(), c.rnd()
        c.put(g * c.nb + 17, a, b, c.pt(c.val(a) + c.val(b)))
        c.put(g * c.nb + 18, a, b, c.pt(-(c.val(a) + c.val(b))), c.rnd())
    q = c.rnd()
    c.put(10 * c.nb + 5, *[q ^ (k & 1) for k in range(200)])
    c.put(12 * c.nb + 1, c.rnd())                                              # a group with only bucket 1: U + S doubles
    c.fill(300, groups=[g for g in range(64) if g not in (3, 10, 12, 31, 63)])
    return c


CASE_FNS = {
    "acc-deep": case_acc_deep,
    "cap-boundary": case_cap_boundary,
    "segments": case_segments,
    "many-heavy": case_many_heavy,
    "reduction-fan3": lambda: case_reduction(3),
    "reduction-fan4": lambda: case_reduction(4),
    "reduction-fan5": lambda: case_reduction(5),
    "group-totals": case_group_totals,
    "tail": lambda: case_tail(True),
    "tail-off": lambda: case_tail(False),
    "prover-2^14": lambda: case_prover(14),
    "prover-2^15": lambda: case_prover(15),
}
_built = {}


def get_case(name):
    if name not in _built:
        _built[name] = CASE_FNS[name]()
    return _built[name]


_sims = {}


def sim_of(name, curve):
    if (name, curve) not in _sims:
        _sims[(name, curve)] = simulate(get_case(name), curve)
    return _sims[(name, curve)]


# ---- CPU: the case table reaches what it claims -----------------------------------------------------------------------------
@pytest.mark.parametrize("curve", ["g1", "g2"])
@pytest.mark.parametrize("name", list(CASE_FNS))
def test_case_reaches_its_branches(name, curve):
    c = get_case(name)
    sim = sim_of(name, curve)
    missing = {e for e in c.expect if sim["events"][e] == 0}
    assert not missing, (name, curve, missing, sim["events"])
    # the model's totals are the weighted sums of its buckets, so its order of operations loses nothing
    for g in range(c.n_groups):
        exp = sum((b + 1) * (sim["buckets"][g * c.nb + b] or 0) for b in range(c.nb)) % R
        assert (sim["totals"][g] or 0) == exp, (name, g)
    for key, lst in c.lists.items():
        assert (sim["buckets"][key] or 0) == sum(c.val(e) or 0 for e in lst) % R, (name, key)


def test_every_event_is_reached_on_both_curves():
    for curve in ("g1", "g2"):
        seen = {e for name in CASE_FNS for e, n in sim_of(name, curve)["events"].items() if n}
        assert seen == set(EVENTS), (curve, set(EVENTS) - seen)


def test_case_shapes():
    """The shapes the cases are named after: a list of exactly cap entries and one of cap + 1, the segment boundaries, more than
    256 heavy buckets, 3 x 64 keys, nb >= 512 with the tail."""
    c = get_case("cap-boundary")
    cap, seg = plan(c)
    assert (cap, seg) == (128, 2048) and c.counts[:2] == [128, 129]
    assert simulate(c, "g1")["heavy"] == 3
    c = get_case("segments")
    assert plan(c) == (128, 2048) and c.counts[:7] == [2047, 2048, 2049, 4096, 4096, 4096, 4196]
    c = get_case("many-heavy")
    assert simulate(c, "g2")["heavy"] == 300 and plan(c)[0] == 128
    assert get_case("acc-deep").n_keys % 128 != 0
    assert simulate(get_case("tail"), "g1")["tail"] and not simulate(get_case("tail-off"), "g1")["tail"]
    assert simulate(get_case("tail-off"), "g1")["levels"] == 3
    assert simulate(get_case("prover-2^15"), "g2")["levels"] == 5


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def knobs(monkeypatch):
    for k in ("OG_RED_FAN0", "OG_MSM_TAIL"):
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def table_points(ctx, curve, logs):
    gen = ctx.g1_generator_mul if curve == "g1" else ctx.g2_generator_mul
    return gen(cport.frs(logs))


def fixed(curve, ds):
    f = cport.g1_fixed_mul_batch if curve == "g1" else cport.g2_fixed_mul_batch
    return f(GEN[curve], cport.frs([d or 0 for d in ds]))


def run_case(ctx, c, curve, buckets):
    ctx.profile(True)
    try:
        ctx.profile_dump()
        tot, bk = ctx.msm_bucket_sums(curve, table_points(ctx, curve, c.logs), c.counts, c.entries, c.n_groups, c.nb,
                                      c.n_entries_max, c.few_groups, buckets)
        prof = ctx.profile_dump()
    finally:
        ctx.profile(False)
    return tot, bk, {k: v[0] for k, v in prof.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["g1", "g2"])
@pytest.mark.parametrize("name", list(CASE_FNS))
def test_bucket_stage_vs_oracle(ctx, knobs, name, curve):
    c = get_case(name)
    if c.fan0:
        knobs.setenv("OG_RED_FAN0", str(c.fan0))
    if not c.tail:
        knobs.setenv("OG_MSM_TAIL", "0")
    sim = sim_of(name, curve)
    tot, bk, prof = run_case(ctx, c, curve, c.buckets)
    pb = PB[curve]
    assert tot == fixed(curve, sim["totals"]), name
    if c.buckets:
        keys = sorted(c.lists)
        got = b"".join(bk[pb * k:pb * k + pb] for k in keys)
        assert got == fixed(curve, [sim["buckets"][k] for k in keys]), name
        empty = [k for k in range(c.n_keys) if k not in c.lists]
        assert all(bk[pb * k:pb * k + pb] == bytes(pb) for k in empty), name
    assert prof.get(f"k_bucket_acc_{curve}") == 1 and prof.get("k_heavy_plan") == 1 and prof.get("k_bucket_order") == 1, prof
    assert prof.get(f"k_bucket_heavy_{curve}") == 1 and prof.get("k_heavy_combine<F>") == 1, prof     # launched on every call
    assert prof.get(f"k_reduce_level_{curve}", 0) == sim["levels"], (sim["levels"], prof)
    assert prof.get(f"k_tail_sums_{curve}", 0) == prof.get(f"k_tail_finish_{curve}", 0) == int(sim["tail"]), prof
    assert prof.get("k_group_total<F>", 0) == int(not sim["tail"]), prof


@pytest.mark.gpu
@pytest.mark.parametrize("curve", ["g1", "g2"])
def test_bucket_stage_reproduces_itself(ctx, knobs, curve):
    """The same lists twice give the same bytes (bucket order and the heavy plan use atomics)."""
    c = get_case("segments")
    a = run_case(ctx, c, curve, True)[:2]
    assert run_case(ctx, c, curve, True)[:2] == a


def _raw(ctx, g2, pts, n_points, counts, entries, n_groups, nb, n_max, few=0):
    cnt = (C.c_uint32 * len(counts))(*counts)
    ent = (C.c_uint32 * max(1, len(entries)))(*entries)
    out = C.create_string_buffer(128 * max(1, n_groups))
    return api.lib().og_msm_bucket_sums(ctx._h, g2, pts, n_points, cnt, ent, n_groups, nb, n_max, few, out, None)


def _last_error(ctx):
    return api.lib().og_last_error(ctx._h).decode(errors="replace")


@pytest.mark.gpu
@pytest.mark.parametrize("g2", [0, 1])
def test_bucket_sums_argument_errors(ctx, g2):
    """Every argument check refuses with OG_E_INVALID before anything is launched."""
    pts = table_points(ctx, "g2" if g2 else "g1", [5, 7])
    E = api.OG_E_INVALID
    n0 = ctx.launch_count
    for nb in (0, 1, 3, 6, 1 << 16, 1 << 17):
        assert _raw(ctx, g2, pts, 2, [0] * (2 * max(nb, 1)), [], 2, nb, 0) == E, nb
    assert _raw(ctx, g2, pts, 2, [1, 1], [2, 4], 1, 2, 2) == E                        # index 2 with two points
    assert _raw(ctx, g2, pts, 2, [1, 1], [2, 5], 1, 2, 2) == E                        # negated, still out of range
    assert _raw(ctx, g2, pts, 2, [2, 0], [0, 3], 1, 2, 1) == E                        # n_entries_max < sum(counts)
    assert _raw(ctx, g2, pts, 2, [2, 0], [0, 3], 1, 2, 1 << 32) == E                  # n_entries_max beyond 32 bits
    assert _raw(ctx, g2, pts, 2, [1 << 31, 1 << 31], [], 1, 2, 1 << 32) == E          # sum(counts) does not fit 32 bits
    assert _raw(ctx, g2, pts, 2, [0, 0], [], 0, 2, 0) == E                            # no groups
    assert _raw(ctx, 2, pts, 2, [0, 0], [], 1, 2, 0) == E
    # n_entries_max whose 4 * avg leaves 32 bits: cap and seg would wrap to 0 (2^31) or 8 (2^31 + 4).  The entry list holds an
    # out-of-range index as well, so the message shows which check refused the call.
    for n_max, counts in ((1 << 31, [1, 0]), ((1 << 31) + 4, [1000, 0]), (1 << 30, [1, 0])):
        assert _raw(ctx, g2, pts, 2, counts, [4], 1, 2, n_max) == E, n_max
        assert "n_entries_max" in _last_error(ctx), (n_max, _last_error(ctx))
    # avg = 512 over 4 x 2^15 keys: cap = seg = 2048, and 32 815 lists of 2049 entries take 65 630 segments, more than the 65 600
    # segment sums the level scratch holds (sum(counts) <= n_entries_max holds)
    n_keys = 4 << 15
    counts = [2049] * 32815 + [0] * (n_keys - 32815)
    assert sum(counts) <= 513 * n_keys - 1
    assert _raw(ctx, g2, pts, 2, counts, [4], 4, 1 << 15, 513 * n_keys - 1) == E
    assert "heavy segments" in _last_error(ctx), _last_error(ctx)
    assert ctx.launch_count == n0
    assert _raw(ctx, g2, pts, 2, [2, 0], [0, 3], 1, 2, 2) == api.OG_OK                 # the boundaries themselves are accepted
    assert _raw(ctx, g2, pts, 2, [2, 0], [0, 3], 1, 2, (1 << 30) - 1) == api.OG_OK
    assert ctx.launch_count > n0
