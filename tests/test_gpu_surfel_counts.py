"""The launch shapes that change with the NUMBER of surfels, past the sizes of the scene tests.

* End tasks (lifecycle.cu LaunchObservationStats): the tile length of ObservationStatsKernel is 32, 64, 128 or 256 surfels,
  picked from N against the resident warps.  ptxas reports 46 registers for the kernel on sm_90a, so 5 CTAs of 256 threads
  fit on an SM: 40 warps per SM, 5,280 on 132 SMs.  The launcher keeps halving the tile (shift 8 -> 5) while the tile count
  is below 1.5 x the resident warps, so on 132 SMs shift 8 needs N >= 256 * 7,920 = 2,027,520, shift 7 N >= 1,013,760 and
  shift 6 N >= 506,880:  24 k -> 32-surfel tiles, 600 k -> 64, 1.2 M -> 128, 2.4 M / 4.2 M / 8.4 M -> 256.  The launcher takes
  the occupancy from cudaOccupancyMaxActiveBlocksPerMultiprocessor (5 on an H100 for this build) and does not report its
  choice, so the figures printed here are this derivation.  A change of the kernel's register count moves the thresholds: at
  40 registers (6 CTAs per SM) every size falls one tile length lower.
* Compaction (CompactScanBlocksKernel): one block sum per 4,096 surfels, scanned in chunks of 1,024 block sums with a carry
  between chunks.  N > 4,194,304 needs a second chunk (4.2 M: 1,026 blocks), 8.4 M a third (2,051 blocks).
* PCG vector kernels (pcg.cu PcgInit2 / Step2 / Step3): grid-stride loops over min(8 x SMs, 2048) blocks of 256 threads,
  i.e. 270,336 unknowns per pass on 132 SMs.  `many` tiled 1, 4 and 8 times has 72,216, 288,216 and 576,216 unknowns:
  one pass, a second partial pass and three passes.

Every expectation here is a restatement: the end-task decision of a surfel depends on that surfel and the keyframes only (the
replicated map repeats the 24 k decisions, which test_gpu_lifecycle pins against the reference), the compaction is a
permutation given by a few lines of numpy, and the PCG vector steps are fp64 axpys and dot products."""
import copy
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DELETED = np.uint32(0x7fffffff)
SCAN_BLOCK = 4096                 # surfels per block sum of the compaction scan
SCAN_CHUNK = 1024 * SCAN_BLOCK    # surfels per chunk of CompactScanBlocksKernel
STATS_CTAS_PER_SM = 5             # ObservationStatsKernel: 46 registers x 256 threads (ptxas -v, sm_90a)


@pytest.fixture(scope="module")
def mods():
    import torch
    assert torch.cuda.is_available()
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    return S, DirectBA, torch


@pytest.fixture(scope="module")
def many_displaced(mods):
    S, _, _ = mods
    return S.displace_surfels(S.make_scene(S.config_by_name("many")))[0]


def stats_tile_shift(n, sm_count):
    """LaunchObservationStats's choice of tile length (lifecycle.cu), with the occupancy of the sm_90a build."""
    warps = STATS_CTAS_PER_SM * sm_count * 8
    shift = 8
    while shift > 5 and 2 * ((n + (1 << shift) - 1) >> shift) < 3 * warps:
        shift -= 1
    return shift


def compaction_sources(deleted):
    """CompactSurfelsCUDAKernel (kernel_compact_surfels.cu:126-157, lifecycle.cu CompactMove*Kernel): the r-th valid surfel
    counted from the end moves into the r-th free slot counted from the front when that slot lies in front of it.  Returns,
    for every slot of the compacted map, the index of the surfel it holds."""
    n = deleted.size
    free = np.flatnonzero(deleted)
    valid_from_end = np.flatnonzero(~deleted)[::-1]
    m = min(free.size, valid_from_end.size)
    f, v = free[:m], valid_from_end[:m]
    moves = f < v
    src = np.arange(n)
    src[f[moves]] = v[moves]
    return src[:n - free.size]


def replicated_scene(sc, R):
    """`sc`'s surfels tiled R times, bit for bit, with row 5 (colour: the end tasks never read it, the compaction moves it)
    replaced by the tag replica * n + original column."""
    n = sc.num_surfels
    N = R * n
    rows = np.tile(sc.surfels[:8, :n], (1, R))
    rows[5] = np.arange(N, dtype=np.uint32).view(np.float32)
    out = copy.copy(sc)
    out.num_surfels = N
    out.surfels = np.zeros((sc.surfels.shape[0], (N + 127) // 128 * 128), np.float32)
    out.surfels[:8, :N] = rows
    return out


@pytest.fixture(scope="module")
def end_task_decisions(mods, many_displaced):
    """Deletion decision and new radius^2 of every original `many` surfel, from the 24 k run."""
    S, DirectBA, _ = mods
    sc = replicated_scene(many_displaced, 1)
    n = sc.num_surfels
    ba = DirectBA.from_scene(sc)
    deleted_count, size = ba.PerformBASchemeEndTasks()
    out = ba.GetSurfelsHost()
    ba.close()
    tags = out[5].view(np.uint32)
    deleted = np.ones(n, bool)
    deleted[tags] = False
    r2 = np.zeros(n, np.float32)
    r2[tags] = out[4]
    assert deleted.sum() == deleted_count > 0 and size == n - deleted_count
    return deleted, r2


@pytest.mark.parametrize("R", [1, 25, 50, 100, 175, 350])
def test_end_tasks_replicated_map(mods, many_displaced, end_task_decisions, R):
    """PerformBASchemeEndTasks on the `many` map tiled R times: every replica gets the decisions of the original surfels, and
    the survivors land where the compaction permutation puts them."""
    S, DirectBA, torch = mods
    deleted1, r2_1 = end_task_decisions
    sc = replicated_scene(many_displaced, R)
    N = sc.num_surfels
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"R={R}: {N} surfels, {sms} SMs -> {1 << stats_tile_shift(N, sms)}-surfel tiles, "
          f"{-(-N // SCAN_BLOCK)} scan blocks in {-(-N // SCAN_CHUNK)} chunk(s)")
    expected = sc.surfels[:8, :N].copy()
    deleted = np.tile(deleted1, R)
    expected[0, deleted] = DELETED.view(np.float32)
    expected[4, ~deleted] = np.tile(r2_1, R)[~deleted]
    src = compaction_sources(deleted)
    expected = expected[:, src]

    ba = DirectBA.from_scene(sc)
    d, size = ba.PerformBASchemeEndTasks()
    assert d == R * int(deleted1.sum()) and size == N - d == ba.surfels_size() == src.size
    out = ba.GetSurfelsHost()
    ba.close()
    assert out.shape == expected.shape
    bad = np.flatnonzero((out.view(np.uint32) != expected.view(np.uint32)).any(axis=0))
    assert bad.size == 0, f"{bad.size} slots differ, first {bad[:5]}: tags {out[5, bad[:5]].view(np.uint32)}, expected {src[bad[:5]]}"


def _pattern(name, n, rng):
    d = np.zeros(n, bool)
    if name == "first":
        d[0] = True
    elif name == "straddle":                          # across the chunk boundary and several 4096-surfel blocks
        d[max(0, SCAN_CHUNK - 3 * SCAN_BLOCK - 17):SCAN_CHUNK + 2 * SCAN_BLOCK + 5] = True
    elif name == "last_chunk":
        start = (n - 1) // SCAN_CHUNK * SCAN_CHUNK
        d[start:] = rng.random(n - start) < 0.1
    elif name == "all_but_last":
        d[:-1] = True
    elif name == "all":
        d[:] = True
    elif name == "random1":
        d = rng.random(n) < 0.01
    elif name == "random50":
        d = rng.random(n) < 0.5
    return d


@pytest.mark.parametrize("n", [SCAN_CHUNK, SCAN_CHUNK + 1, 8_400_000])
def test_compact_surfels_across_scan_chunks(mods, n):
    """bba_compact_surfels on synthetic deletion patterns at 1,024 / 1,025 / 2,051 scan blocks, with and without the active
    flags, against the numpy permutation.  Every surfel's eight rows hold 8 * index + row, so each slot names its source."""
    S, DirectBA, torch = mods
    from badslam_b200.direct_ba import PinholeCamera4f
    dev = torch.device("cuda", torch.cuda.current_device())
    pitch = (n + 127) // 128 * 128
    cam = PinholeCamera4f(64, 48, [30, 30, 32, 24])
    ba = DirectBA(pitch, 1e-3, 40, 4, color_camera_initial_estimate=cam, depth_camera_initial_estimate=cam)   # (no keyframes)
    idx = torch.arange(n, device=dev, dtype=torch.int64)
    base = (idx[None, :] * 8 + torch.arange(8, device=dev)[:, None]).to(torch.int32)
    base_active = ((idx * 37 + 11) & 0xff).to(torch.uint8)
    rng = np.random.default_rng(n)
    for name in ["first", "straddle", "last_chunk", "all_but_last", "all", "random1", "random50"]:
        deleted = _pattern(name, n, rng)
        free = int(deleted.sum())
        src = compaction_sources(deleted)
        src_t = torch.from_numpy(src).to(dev)
        for with_active in (False, True):
            surf = torch.zeros((17, pitch), dtype=torch.float32, device=dev)
            surf.view(torch.int32)[:8, :n] = base
            surf[0, :n][torch.from_numpy(deleted).to(dev)] = torch.tensor(int(DELETED), dtype=torch.int32).view(torch.float32)
            active = torch.zeros(pitch, dtype=torch.uint8, device=dev)
            active[:n] = base_active
            ba.SetSurfels(surf, n, active)
            assert ba.CompactSurfels(free, with_active) == n - free == src.size
            torch.cuda.synchronize()
            m = src.size
            got = surf.view(torch.int32)[:8, :m]
            ok = torch.equal(got, base[:, src_t]) if m else True
            assert ok, (name, with_active, int((got != base[:, src_t]).any(dim=0).nonzero()[0, 0]))
            if with_active:
                assert torch.equal(active[:m], base_active[src_t]), (name, "active flags")
            else:
                assert torch.equal(active[:n], base_active), (name, "active flags touched")
            if name == "first":   # the last surfel, past the first scan chunk when n > 4,194,304, fills slot 0
                assert int(got[0, 0]) == 8 * (n - 1)
    ba.close()


# ---- PCG vector kernels past one grid pass ---------------------------------------------------------------------------------
EPS32 = 2.0 ** -23          # fp32 ulp of 1
GAUGE = 16                  # first keyframe of the second 16-keyframe group
A_INIT = 0.02


def ulps(k, *terms):
    """k fp32 ulps of the sum of the magnitudes of `terms` (element-wise)."""
    return k * EPS32 * sum(np.abs(np.asarray(t, np.float64)) for t in terms)


def pcg_scene(S, R, intr):
    """`many` (with depth-distorted images and perturbed cameras when intrinsics are optimised) with its surfels tiled R
    times.  Every 7th surfel is moved out of every view with descriptors 1 / 2 at +200 / -200: without residuals its steps
    are zero, so the update's clamp to +-180 must bring them back.  (An observed descriptor moves towards what the keyframes
    measure, i.e. inwards, and never reaches the clamp.)"""
    from gpu_checks import distorted_scene
    base = distorted_scene(S, "many") if intr else S.make_scene(S.config_by_name("many"))
    sc = copy.copy(base)
    n = base.num_surfels
    sc.num_surfels = N = R * n
    sc.surfels = np.zeros((base.surfels.shape[0], (N + 127) // 128 * 128), np.float32)
    sc.surfels[:8, :N] = np.tile(base.surfels[:8, :n], (1, R))
    sc.surfels[0, :N:7] += np.float32(1000.0)
    sc.surfels[6, :N:7] = 200.0
    sc.surfels[7, :N:7] = -200.0
    return sc


class Layout:
    """Unknowns of the PCG solver (direct_ba_pcg.cc:273-309): 6 per keyframe but the gauge, 3 per surfel (offset along the
    normal, descriptor 1, descriptor 2), then fx^-1 fy^-1 cx^-1 cy^-1 a + one cfactor per cell and the colour intrinsics."""

    def __init__(self, sc, intr):
        K, N = sc.cfg.num_keyframes, sc.num_surfels
        self.surfel_start = 6 * (K - 1)
        self.depth_start = self.surfel_start + 3 * N
        self.cells = sc.cfactor.size
        self.U = self.depth_start + ((5 + self.cells + 4) if intr else 0)
        self.a_index = self.depth_start + 4 if intr else -1
        self.color_start = self.depth_start + 5 + self.cells
        lam = np.full(self.U, np.float32(1e-8), np.float32)   # kDiagEpsilon, + the prior weight^2 on `a` (pcg.cu DiagExtra)
        if intr:
            lam[self.a_index] = np.float32(1e-8) + np.float32(100.0)
        self.lam = lam


def fsum_products(a, b):
    """The fp32 products a_i * b_i summed exactly (math.fsum) and the sum of their magnitudes."""
    t = (np.asarray(a, np.float32) * np.asarray(b, np.float32)).astype(np.float64)
    return math.fsum(t.tolist()), math.fsum(np.abs(t).tolist())


# GridOrderedAdd sums fp64 partials: per thread over its grid-stride elements (<= 3 here), a warp and a block tree (13 levels),
# then the <= 2048 block partials in order.  Every term here is >= 0 (r^2 / (M + lambda), lambda p^2), so the result is within
# ~(3 + 13 + 2048) * 2^-53 < 3e-13 of the exact sum relative to the sum; 1e-12 leaves room and still catches one missing element.
SUM_REL = 1e-12


def check_step(L, s, K, a):
    """Restates PCGInit2 (for step 0), PCGStep2 and PCGStep3 in fp64 from the kernel's own inputs of the same call."""
    lam, U = L.lam, L.U
    r, M, p, g, delta = (s[k] for k in ("r", "M", "p", "g", "delta"))
    assert all(s[k].shape == (U,) for k in ("r", "M", "p", "g", "delta", "r_step2", "delta_step2", "z", "p_step3", "g_step3"))
    denom = M + lam                                  # fp32 add, as in the kernel
    if s["step"] == 0:
        # PCGInit2: p = r' / (M + lambda), r' = r with the prior on `a`; fast-math division: <= 2 ulps, 4 allowed
        r_prior = r.copy()
        if L.a_index >= 0:
            r_prior[L.a_index] = r[L.a_index] + np.float32(-100.0) * np.float32(a)
        p_expected = r_prior.astype(np.float64) / denom
        err = np.abs(p - p_expected)
        assert np.all(err <= ulps(4, p_expected)), ("init2 p", int(np.argmax(err - ulps(4, p_expected))))
        # alpha_n = sum fl32(r' p) in fp64; the prior's product and add may be one FMA: one ulp of the `a` term more
        exact, mag = fsum_products(r_prior, p)
        extra = ulps(1, r_prior[L.a_index] * np.float64(p[L.a_index])) if L.a_index >= 0 else 0.0
        assert abs(s["alpha_n"] - exact) <= SUM_REL * mag + extra, ("init2 alpha_n", s["alpha_n"], exact)
        # alpha_d = K sum fl32(fl32(lambda p) p) + p^T J^T W J p (PCGStep1).  The second part is an fp32 sum per item, g an fp32
        # atomic sum per entry (up to ~10^4 terms: ~10^4 * 2^-24 ~ 6e-4 relative): they agree to 1e-3 of sum |p_i g_i|
        lam_part, _ = fsum_products(lam * p, p)
        pg = np.asarray(p, np.float64) * g
        assert abs((s["alpha_d"] - K * lam_part) - math.fsum(pg.tolist())) <= 1e-3 * math.fsum(np.abs(pg).tolist()), "alpha_d vs p.g"
    # PCGStep2: alpha = fl32(alpha_n) / fl32(alpha_d) (fast-math: <= 2 ulps); each element is one or two FMAs on top
    alpha = np.float64(np.float32(s["alpha_n"])) / np.float64(np.float32(s["alpha_d"]))
    d_exp = delta + alpha * p
    err = np.abs(s["delta_step2"] - d_exp)
    assert np.all(err <= ulps(4, delta, alpha * p)), ("step2 delta", int(np.argmax(err - ulps(4, delta, alpha * p))))
    r_exp = r - alpha * (g + lam.astype(np.float64) * p)
    tol = ulps(4, r, alpha * g, alpha * lam * p.astype(np.float64))
    err = np.abs(s["r_step2"] - r_exp)
    assert np.all(err <= tol), ("step2 r", int(np.argmax(err - tol)))
    z_exp = s["r_step2"].astype(np.float64) / denom
    err = np.abs(s["z"] - z_exp)
    assert np.all(err <= ulps(4, z_exp)), ("step2 z", int(np.argmax(err - ulps(4, z_exp))))
    exact, mag = fsum_products(s["z"], s["r_step2"])
    assert abs(s["beta_n"] - exact) <= SUM_REL * mag, ("step2 beta_n", s["beta_n"], exact)
    # PCGStep3: beta = fl32(beta_n) / fl32(alpha_n), p = z + beta p (one FMA), g cleared, alpha_d re-armed with K sum lambda p^2
    beta = np.float64(np.float32(s["beta_n"])) / np.float64(np.float32(s["alpha_n"]))
    p3 = s["z"] + beta * p
    err = np.abs(s["p_step3"] - p3)
    assert np.all(err <= ulps(4, s["z"], beta * p)), ("step3 p", int(np.argmax(err - ulps(4, s["z"], beta * p))))
    assert not np.any(s["g_step3"]), "step3 g"
    lam_part, mag = fsum_products(lam * s["p_step3"], s["p_step3"])
    assert abs(s["alpha_d_step3"] - K * lam_part) <= SUM_REL * K * mag, ("step3 alpha_d", s["alpha_d_step3"], K * lam_part)


def check_apply(S, L, sc, before, after, delta, intr):
    """The solver's update from pcg_delta (direct_ba_pcg.cc:552-638)."""
    K, N = sc.cfg.num_keyframes, sc.num_surfels
    rows0, rows1 = before["surfels"], after["surfels"]
    su = L.surfel_start + 3 * np.arange(N)
    t = delta[su].astype(np.float64)
    nrm = S.unpack_surfel_normal(rows0[3].view(np.uint32)).astype(np.float64)
    x_exp = rows0[:3].astype(np.float64) + t[None, :] * nrm.T
    # x += t n: one rounding of the sum (1 ulp of x) plus |t| times the precision of the device's unpacked normal (rsqrt
    # normalisation under fast math: a few fp32 ulps of a unit vector; 8 allowed)
    tol = np.spacing(np.abs(x_exp).astype(np.float32)) + np.abs(t)[None, :] * 8 * EPS32
    err = np.abs(rows1[:3] - x_exp)
    assert np.all(err <= tol), ("x += t n", np.unravel_index(np.argmax(err - tol), err.shape))
    assert np.array_equal(rows1[3:6].view(np.uint32), rows0[3:6].view(np.uint32))
    # descriptors: clamp(d + delta, +-180) in fp32, bit for bit; the clamp must have fired on the unobserved surfels
    for row, off, bound in ((6, 1, 180.0), (7, 2, -180.0)):
        raw = rows0[row] + delta[su + off]
        assert np.array_equal(rows1[row].view(np.uint32), np.clip(raw, np.float32(-180), np.float32(180)).view(np.uint32)), row
        assert np.all(rows1[row][::7] == np.float32(bound)), ("clamp", row)
    # poses: global_T_frame o Exp(delta) for every keyframe but the gauge; host fp32 SE3 arithmetic: a few ulps of translations
    # of up to ~3 m (ulp 2.4e-7) and of the unit quaternion
    for k in range(K):
        if k == GAUGE:
            assert np.array_equal(after["poses"][k], before["poses"][k])
            continue
        j = 6 * (k if k < GAUGE else k - 1)
        exp = S.se3_mul(before["poses"][k], S.se3_exp(delta[j:j + 6]))
        dt, dr = S.pose_error(after["poses"][k], exp)
        assert dt < 2e-6 and dr < 2e-6, (k, dt, dr)
    d0, c0, a0 = before["intr"]
    d1, c1, a1 = after["intr"]
    if intr:
        di, ci = delta[L.depth_start:L.depth_start + 5], delta[L.color_start:L.color_start + 4]
        # cfactor += delta and a += delta_a: fp32 adds, bit for bit
        assert np.array_equal(after["cfactor"].reshape(-1), before["cfactor"].reshape(-1) + delta[L.depth_start + 5:L.depth_start + 5 + L.cells])
        assert np.float32(a1) == np.float32(a0) + di[4]
        # depth intrinsics through the inverse parametrisation in double (direct_ba_pcg.cc:590-612), then rounded to fp32
        fx_inv, fy_inv = 1.0 / np.float64(d0[0]), 1.0 / np.float64(d0[1])
        cx_inv, cy_inv = -(np.float64(d0[2]) - 0.5) * fx_inv, -(np.float64(d0[3]) - 0.5) * fy_inv
        fx, fy = 1.0 / (fx_inv + np.float64(di[0])), 1.0 / (fy_inv + np.float64(di[1]))
        d_exp = np.array([fx, fy, -(fx * (cx_inv + np.float64(di[2]))) + 0.5, -(fy * (cy_inv + np.float64(di[3]))) + 0.5])
        assert np.all(np.abs(d1 - d_exp) <= np.spacing(np.abs(d_exp).astype(np.float32))), (d1, d_exp)
        assert np.array_equal(c1, (c0 + ci).astype(np.float32)), (c1, c0 + ci)
        assert np.any(d1 != d0) and np.any(after["cfactor"] != before["cfactor"])
    else:
        assert np.array_equal(d1, d0) and np.array_equal(c1, c0) and a1 == a0
        assert np.array_equal(after["cfactor"], before["cfactor"])


def handle_state(ba):
    return {"surfels": ba.GetSurfelsHost(), "poses": ba.GetKeyframeStates()[0].copy(), "intr": ba._intrinsics(),
            "cfactor": ba.cfactor_buffer()}


def probe(ba, step, intr, apply=False):
    s = ba.PCGProbe(step, apply, optimize_depth_intrinsics=intr, optimize_color_intrinsics=intr, gauge_keyframe=GAUGE)
    s["step"] = step
    return s


def pcg_handle(S, DirectBA, sc, intr):
    ba = DirectBA.from_scene(sc)
    if intr:   # a non-zero deformation model: the prior term on `a` and the d/da, d/dcfactor Jacobians are live
        ba.SetA(A_INIT)
        ba.SetCFactorBuffer((np.random.default_rng(5).standard_normal(sc.cfactor.shape) * 0.003).astype(np.float32))
    return ba


@pytest.mark.parametrize("intr", [False, True])
@pytest.mark.parametrize("R", [1, 4, 8])
def test_pcg_vector_steps_across_grid_passes(mods, R, intr):
    """PCGInit2, two inner steps (PCGStep2 / PCGStep3 in both scalar-slot orders) and the update, at 1, 2 (partial) and 3 grid
    passes of the vector kernels, against fp64 restatements from the kernels' own inputs."""
    S, DirectBA, torch = mods
    sc = pcg_scene(S, R, intr)
    L = Layout(sc, intr)
    K = sc.cfg.num_keyframes
    ba = pcg_handle(S, DirectBA, sc, intr)
    a = ba._intrinsics()[2]
    threads = 256 * min(8 * torch.cuda.get_device_properties(0).multi_processor_count, 2048)
    print(f"R={R} intrinsics={intr}: {L.U} unknowns, {-(-L.U // threads)} grid pass(es)")
    s0 = probe(ba, 0, intr)
    assert s0["r"].size == L.U
    check_step(L, s0, K, a)
    before = handle_state(ba)
    s1 = probe(ba, 1, intr, apply=True)
    check_step(L, s1, K, a)
    check_apply(S, L, sc, before, handle_state(ba), s1["delta_step2"], intr)


def test_pcg_vector_steps_large_then_small_on_one_handle(mods):
    """Three grid passes, then one on the same handle: ordered-sum partials or arrival counters left behind by the larger
    launch would corrupt the smaller one's dot products."""
    S, DirectBA, torch = mods
    big, small = pcg_scene(S, 8, True), pcg_scene(S, 1, True)
    ba = pcg_handle(S, DirectBA, big, True)
    a = ba._intrinsics()[2]
    K = big.cfg.num_keyframes
    for sc in (big, small):
        if sc is small:
            ba.SetSurfels(torch.from_numpy(small.surfels).cuda(), small.num_surfels)
        L = Layout(sc, True)
        s = probe(ba, 1, True)
        assert s["r"].size == L.U
        check_step(L, s, K, a)
