"""The MSM's plan space on the GPU, checked against known discrete logs.

A plan is the window c and the table mode (per table: msm_window_for / table_new in capi.cu), plus the task length and
the reduction chunk (per call: msm_tuning).  Every case builds bases P_i = k_i B on the device (b200_fixed_base_batch)
with 64 of them checked against the big-int oracle, so that a fixed-base error is not blamed on the MSM; the expected
sum is (sum k_i s_i mod r) B, compared in affine form.  Every case asserts the plan it reached through table.info() and
names it in its id or assertion message.  The scalar families are msm_families.py's."""
import numpy as np
import pytest

from msm_families import FAMILIES, pack, seeded, uniform
from oracle import corelib, ec, ff
from oracle.params import CURVES
from util import jac_to_affine, pick_base

pytestmark = pytest.mark.gpu

PAIRS = [(c, g) for c in CURVES.values() for g in (1, 2)]
PAIR_IDS = [f"{c.name}-g{g}" for c, g in PAIRS]
BY_NAME = dict(zip(PAIR_IDS, PAIRS))
MAX_WINDOWS = 64          # MSM_MAX_WINDOWS of the table precompute (msm_impl.cuh)
N_SWEEP = 3000            # not a multiple of 128 or 256


def coord_limbs(curve, group):
    return curve.fp_limbs * (curve.g2_degree if group == 2 else 1)


def effective_window(curve, c):
    """table_new: c grows until the scalar has at most 64 windows"""
    while curve.r.bit_length() // c + 1 > MAX_WINDOWS:
        c += 1
    return c


def default_window(curve, n):
    """msm_window_for without an override: floor(log2 n) - 4, clamped to [4, 16]"""
    return effective_window(curve, min(16, max(4, n.bit_length() - 1 - 4)))


def need_free(gib, what):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < gib * 2 ** 30:
        pytest.skip(f"{what} needs about {gib} GiB of free device memory; {free / 2 ** 30:.1f} GiB free, "
                    f"{gib - free / 2 ** 30:.1f} GiB short")


def build_bases(gpu, curve, group, n, key):
    """(F, B, ks, d_pts): ks (n, fr_limbs) Montgomery discrete logs, d_pts the n points k_i B on the device"""
    import torch
    F, B = pick_base(curve, group)
    ks = uniform(curve, n, seeded("bases", key))
    d_ks = torch.from_numpy(ks.view(np.int64)).cuda()
    d_pts = torch.zeros((n, 2 * coord_limbs(curve, group)), dtype=torch.int64, device="cuda")
    gpu.fixed_base_batch(curve.curve_id, group, ec.pack_points(curve, group, [B]), d_ks, n=n, out=d_pts)
    del d_ks
    rng = seeded("spot", key)
    idx = sorted({0, n - 1} | {rng.randrange(n) for _ in range(62)})
    pts = ec.unpack_points(curve, group, d_pts[idx].cpu().numpy().view(np.uint64))
    kv = ff.unpack_elements(ks[idx], curve.r, curve.fr_limbs)
    for i, P_, k in zip(idx, pts, kv):
        assert P_ == ec.scalar_mul(F, k, B), f"fixed-base batch: base {i} of {curve.name} G{group} is not k_i B"
    return F, B, ks, d_pts


_BASES = {}
N_CACHED = (1 << 20) + 1     # the largest table of the default-window sizes


def bases(gpu, curve, group):
    """N_CACHED known-discrete-log bases per curve and group, built once per session"""
    key = (curve.name, group)
    if key not in _BASES:
        _BASES[key] = build_bases(gpu, curve, group, N_CACHED, key)
    return _BASES[key]


def make_table(gpu, curve, group, n, precomp, start=0):
    F, B, ks, d_pts = bases(gpu, curve, group)
    t = gpu.Table(curve.curve_id, group, d_pts[start:start + n], precomp=precomp, n=n, on_device=True)
    return t, ks[start:start + n]


def plan_of(t, curve, group):
    i = t.info()
    return i, f"{curve.name} G{group} n={i['n']} c={i['window_bits']} windows={i['n_windows']} precomp={i['precomp']}"


def assert_plan(t, curve, group, c, precomp):
    info, plan = plan_of(t, curve, group)
    assert (info["window_bits"], info["n_windows"], info["precomp"]) == (c, curve.r.bit_length() // c + 1, int(precomp)), plan
    return plan


def expected(curve, group, ks, sc):
    F, B = pick_base(curve, group)
    return ec.scalar_mul(F, corelib.fr_dot(curve, ks, sc), B)


def check_msm(t, curve, group, ks, sc, what, off=0):
    """MSM of sc against the bases [off, off + len(sc)) of t, against the known discrete logs ks of those bases"""
    n = sc.shape[0]
    got = jac_to_affine(curve, group, t.msm(sc, off=off, n=n))
    assert got == expected(curve, group, ks[off:off + n], sc), what
    return got


# ---- (a) every window, every family ---------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("c", range(4, 21), ids=lambda c: f"c{c}")
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_window_sweep(gpu, monkeypatch, pair, c, precomp):
    """GB200_MSM_WINDOW = c on a table of N_SWEEP bases; BW6-761 (377-bit scalars) raises c = 4, 5 to 6 so that the
    precompute's 64 windows suffice.  Includes the windows that divide the scalar length (an extra, carry-only top
    window: 255 at c = 5, 15; 253 at 11; 377 at 13) and the windows that leave c - 1 bits on top."""
    curve, group = BY_NAME[pair]
    eff = effective_window(curve, c)
    if curve.name == "bw6-761":
        assert eff == (6 if c < 6 else c)
    monkeypatch.setenv("GB200_MSM_WINDOW", str(c))
    t, ks = make_table(gpu, curve, group, N_SWEEP, precomp)
    plan = assert_plan(t, curve, group, eff, precomp)
    for fam in FAMILIES:
        sc = pack(curve, eff, fam, N_SWEEP, seeded("sweep", pair, c, fam))
        check_msm(t, curve, group, ks, sc, f"{plan} family={fam}")
    t.free()


# ---- (b) the default window --------------------------------------------------------------------------------------------
DEFAULT_SIZES = sorted({1 << k for k in range(8, 21)} | {(1 << k) + d for k in range(9, 21) for d in (-1, 1)})


@pytest.mark.parametrize("n", DEFAULT_SIZES)
@pytest.mark.parametrize("pair", ["bn254-g1", "bn254-g2", "bls12-381-g2", "bw6-761-g1"])
def test_default_window(gpu, monkeypatch, pair, n):
    """c = clamp(floor(log2 n) - 4, 4, 16) at 2^8..2^20 bases and on both sides of every size where c changes;
    powers of two on plain tables, the sizes next to them on precomputed ones"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    precomp = n & (n - 1) != 0
    t, ks = make_table(gpu, curve, group, n, precomp)
    c = default_window(curve, n)
    plan = assert_plan(t, curve, group, c, precomp)
    for fam in ("uniform", "mixed"):
        check_msm(t, curve, group, ks, pack(curve, c, fam, n, seeded("default", pair, n, fam)), f"{plan} family={fam}")
    t.free()


# ---- (c) sub-ranges of precomputed tables ------------------------------------------------------------------------------
@pytest.mark.parametrize("c", (12, 13, 16), ids=lambda c: f"c{c}")
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_precomputed_subranges(gpu, monkeypatch, pair, c):
    """slab index w * stride + off + i with off > 0: one scalar at the first, a middle and the last base, and a range
    that ends at the table's end"""
    curve, group = BY_NAME[pair]
    monkeypatch.setenv("GB200_MSM_WINDOW", str(c))
    t, ks = make_table(gpu, curve, group, N_SWEEP, True, start=777)
    plan = assert_plan(t, curve, group, c, True)
    rng = seeded("subrange", pair, c)
    for off in (0, 1234, N_SWEEP - 1):
        for fam in ("uniform", "r_minus_1", "top_window_max"):
            check_msm(t, curve, group, ks, pack(curve, c, fam, 1, rng), f"{plan} off={off} n=1 family={fam}", off=off)
    for off in (1, 1001, N_SWEEP - 129):
        sc = pack(curve, c, "mixed", N_SWEEP - off, rng)
        check_msm(t, curve, group, ks, sc, f"{plan} off={off} n={N_SWEEP - off}", off=off)
    t.free()


# ---- (d) forced task length and chunk ---------------------------------------------------------------------------------
N_TUNE = 1 << 14          # c = 10: 512 buckets per set, ~800 entries per bucket on a precomputed table


@pytest.mark.parametrize("task_len", (1, 2, 7, 64, 1000, 1 << 20, 0, -1))
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", ["bn254-g1", "bls12-381-g2", "bw6-761-g1"])
def test_tuning_overrides(gpu, monkeypatch, pair, precomp, task_len):
    """GB200_MSM_TASK_LEN x GB200_MSM_CHUNK (tools/sweep_msm.py's knobs).  0 and -1 are out of range and must fall
    back to the fitted task length / default chunk: taken as they are, 0 divides by zero in msm_layout and a task
    length of -1 (0xffffffff) wraps the rounded-up task count of every bucket with 2 or more entries to 0.  A chunk of
    2^c is capped at the 2^(c-1) buckets of a set."""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_TUNE, precomp)
    c = default_window(curve, N_TUNE)
    plan = assert_plan(t, curve, group, c, precomp)
    sc = pack(curve, c, "mixed", N_TUNE, seeded("tune", pair, precomp))
    want = expected(curve, group, ks, sc)
    monkeypatch.setenv("GB200_MSM_TASK_LEN", str(task_len))
    for chunk in (1, 3, 1 << (c - 1), 1 << c, 0, -1):
        monkeypatch.setenv("GB200_MSM_CHUNK", str(chunk))
        assert jac_to_affine(curve, group, t.msm(sc)) == want, f"{plan} task_len={task_len} chunk={chunk}"
    t.free()


# ---- (e) heavy buckets -------------------------------------------------------------------------------------------------
N_HEAVY = 1 << 16


@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_heavy_buckets(gpu, monkeypatch, pair, precomp):
    """buckets of thousands of entries = far more than 48 task partials each, which k_msm_combine queues for the warp
    tree of k_msm_combine_heavy (48 KiB of shared memory per block for the 384-byte XYZZ points of BLS12 G2 and
    BW6-761)"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, N_HEAVY, precomp)
    c = default_window(curve, N_HEAVY)
    plan = assert_plan(t, curve, group, c, precomp)
    r = curve.r
    g = np.random.default_rng(seeded("heavy", pair).randrange(1 << 63))
    cand = ff.pack_elements([0, 1, 2, 3, 1 << (c - 1), r - 1], r, curve.fr_limbs)
    pick = np.where(g.random(N_HEAVY) < 0.5, 0, g.integers(1, 6, size=N_HEAVY))
    check_msm(t, curve, group, ks, np.ascontiguousarray(cand[pick]), f"{plan} half zero, rest in {{1, 2, 3, 2^(c-1), r-1}}")
    t.free()


@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_heavy_buckets_equal_bases(gpu, monkeypatch, pair, precomp):
    """every base the same point (groth16.DummySetup): with equal scalars every full task has the same partial sum and
    so does every lane of the warp tree, so the combine step and the tree add a point to itself (XYZZ::add's doubling
    branch); with 1 and r - 1 = -1 mixed in, partial sums also cancel to infinity"""
    import torch
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    F, B, ks, d_pts = bases(gpu, curve, group)
    k0 = ks[5:6]
    d_same = d_pts[5:6].expand(N_HEAVY, -1).contiguous()
    t = gpu.Table(curve.curve_id, group, d_same, precomp=precomp, n=N_HEAVY, on_device=True)
    del d_same
    torch.cuda.synchronize()
    c = default_window(curve, N_HEAVY)
    plan = assert_plan(t, curve, group, c, precomp)
    KS = np.ascontiguousarray(np.repeat(k0, N_HEAVY, axis=0))
    r = curve.r
    ones = ff.pack_elements([1], r, curve.fr_limbs).repeat(N_HEAVY, axis=0)
    check_msm(t, curve, group, KS, np.ascontiguousarray(ones), f"{plan} equal bases, every scalar 1")
    g = np.random.default_rng(seeded("equal", pair).randrange(1 << 63))
    cand = ff.pack_elements([1, r - 1, 1 << (c - 1)], r, curve.fr_limbs)
    sc = np.ascontiguousarray(cand[g.choice(3, size=N_HEAVY, p=(0.45, 0.45, 0.1))])
    check_msm(t, curve, group, KS, sc, f"{plan} equal bases, scalars in {{1, -1, 2^(c-1)}}")
    t.free()


# ---- (f) full size at the default plans ---------------------------------------------------------------------------------
@pytest.mark.parametrize("precomp", (False, True), ids=("plain", "precomp"))
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_full_size(gpu, monkeypatch, pair, precomp):
    """2^20 bases at the default plan (c = 16); on the precomputed table also a few thousand scalars in the middle
    (sparse buckets) and one scalar on the last base"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    need_free(12, f"{pair} 2^20 table")
    n = 1 << 20
    t, ks = make_table(gpu, curve, group, n, precomp)
    c = default_window(curve, n)
    plan = assert_plan(t, curve, group, c, precomp)
    rng = seeded("full", pair, precomp)
    for fam in ("uniform", "mixed"):
        check_msm(t, curve, group, ks, pack(curve, c, fam, n, rng), f"{plan} family={fam}")
    if precomp:
        off = (1 << 19) + 12345
        check_msm(t, curve, group, ks, pack(curve, c, "mixed", 4099, rng), f"{plan} off={off} n=4099", off=off)
        check_msm(t, curve, group, ks, pack(curve, c, "r_minus_1", 1, rng), f"{plan} off={n - 1} n=1", off=n - 1)
    t.free()


@pytest.mark.parametrize("n", ((1 << 18) + 1, 3 * (1 << 18) - 5))
@pytest.mark.parametrize("pair", PAIR_IDS)
def test_precompute_chunk_boundary(gpu, monkeypatch, pair, n):
    """the table precompute works in chunks of 2^18 bases: tables that end one base past a chunk and inside the third"""
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    t, ks = make_table(gpu, curve, group, n, True)
    c = default_window(curve, n)
    plan = assert_plan(t, curve, group, c, True)
    rng = seeded("boundary", pair, n)
    check_msm(t, curve, group, ks, pack(curve, c, "mixed", n, rng), plan)
    for off in (min((1 << 18) - 3, n - 7), n - 7):     # a range across the first chunk boundary, one at the end
        check_msm(t, curve, group, ks, pack(curve, c, "uniform", 7, rng), f"{plan} off={off} n=7", off=off)
    t.free()


def test_bw6_761_g1_2_24_single_gpu(gpu, monkeypatch):
    """BASELINE config 5 on one GPU: BW6-761 G1, 2^24 bases, plain table (about 13 GB of table and workspace)"""
    import torch
    curve, group = CURVES["bw6-761"], 1
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    need_free(20, "BW6-761 G1 2^24")
    n = 1 << 24
    F, B, ks, d_pts = build_bases(gpu, curve, group, n, ("bw6-761", 1, "2^24"))
    t = gpu.Table(curve.curve_id, group, d_pts, precomp=False, n=n, on_device=True)
    del d_pts
    torch.cuda.empty_cache()
    c = default_window(curve, n)
    plan = assert_plan(t, curve, group, c, False)
    check_msm(t, curve, group, ks, pack(curve, c, "mixed", n, seeded("bw6-2^24")), plan)
    t.free()


# ---- (g) the other MSM entry points -------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", ["bn254-g1", "bls12-381-g2", "bls12-377-g1", "bw6-761-g2"])
def test_pipelined_and_profiled(gpu, monkeypatch, pair):
    """b200_msm_pipelined twice back to back, then join; then b200_msm_profile: both equal b200_msm"""
    import torch
    curve, group = BY_NAME[pair]
    monkeypatch.delenv("GB200_MSM_WINDOW", raising=False)
    n = N_TUNE
    t, ks = make_table(gpu, curve, group, n, True)
    c = default_window(curve, n)
    plan = assert_plan(t, curve, group, c, True)
    rng = seeded("entry", pair)
    sc = [pack(curve, c, "mixed", n, rng), pack(curve, c, "uniform", n, rng)]
    want = [check_msm(t, curve, group, ks, s, f"{plan} b200_msm") for s in sc]
    d_sc = [torch.from_numpy(s.view(np.int64)).cuda() for s in sc]
    d_out = torch.zeros((3, 3 * coord_limbs(curve, group)), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    t.msm_pipelined(d_sc[0], d_out[0], n=n)
    t.msm_pipelined(d_sc[1], d_out[1], n=n)
    t.join()
    gpu.sync(0)
    prof = t.msm_profile(d_sc[0], d_out[2], n=n)
    gpu.sync(0)
    out = d_out.cpu().numpy().view(np.uint64)
    assert jac_to_affine(curve, group, out[0]) == want[0], f"{plan} first pipelined MSM"
    assert jac_to_affine(curve, group, out[1]) == want[1], f"{plan} second pipelined MSM"
    assert jac_to_affine(curve, group, out[2]) == want[0], f"{plan} profiled MSM"
    assert set(prof) == set(t.MSM_STAGES) and all(v >= 0 for v in prof.values()), prof
    t.free()
