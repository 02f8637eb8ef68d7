"""The trajectory deformation around a BA call (ExtrapolateAndInterpolateKeyframePoseChanges, trajectory_deformation.cc:45-130):
the library's host function (bba_host_deform_trajectory, its Python and C++ mirrors) against oracle/trajectory_oracle.py, and
both against what the deformation must do by construction.  CPU only."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from badslam_b200 import _lib
from badslam_b200.direct_ba import deform_trajectory
from oracle import cpu_oracle as O
from oracle import trajectory_oracle as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDENT = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)


def random_pose(rng, rot=0.5, trans=2.0):
    return O.se3_exp(np.concatenate([rng.uniform(-trans, trans, 3), rng.uniform(-rot, rot, 3)]).astype(np.float32))


def product(idx, original, current, start, end, frames):
    out = np.array(frames, np.float32, copy=True)
    deform_trajectory(start, end, idx, original, current, out)
    return out


def oracle(idx, original, current, start, end, frames):
    return T.deform_trajectory(idx, original, current, start, end, frames)


IMPLS = {"product": product, "oracle": oracle}


def within_ulps(a, b, n):
    """|a - b| <= n ulps per component, an ulp taken at the component's scale: 1 for the unit quaternion, the larger translation
    component of the two poses for the translation."""
    a, b = np.asarray(a, np.float32).reshape(-1, 7), np.asarray(b, np.float32).reshape(-1, 7)
    scale = np.ones_like(a)
    scale[:, 4:] = np.maximum(np.abs(a[:, 4:]).max(1, keepdims=True), np.abs(b[:, 4:]).max(1, keepdims=True))
    return bool((np.abs(a.astype(np.float64) - b) <= n * np.spacing(scale.astype(np.float32))).all())


def same_pose(a, b, tol):
    """a and b are the same rigid transform to `tol` (q and -q are the same rotation)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if np.dot(a[:4], b[:4]) < 0:
        b = np.concatenate([-b[:4], b[4:]])
    return np.abs(a - b).max() <= tol


def trajectory(rng, n, keyframe_count, bump=0.05):
    """n frame poses, keyframe_count keyframes among frames 3 .. n - 4 (so that frames lie before, between and after them), the
    keyframes' frame_T_global before BA and their poses after it (each moved by its own small random motion)."""
    frames = np.stack([random_pose(rng) for _ in range(n)])
    idx = np.sort(rng.choice(np.arange(3, n - 3), keyframe_count, replace=False)).astype(np.int32)
    original = np.stack([O.se3_inverse(frames[i]) for i in idx])
    current = np.stack([O.se3_mul(random_pose(rng, bump, bump), frames[i]) for i in idx])
    return frames, idx, original, current


@pytest.mark.parametrize("start", [0, 2])
@pytest.mark.parametrize("keyframe_count", [1, 2, 10])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_product_matches_the_oracle(seed, keyframe_count, start):
    """Frames before the first, between and after the last keyframe, from start_frame 0 and 2, to within 2 ulps per component.
    The two evaluate the same fp32 operations in the same order (Sophus products, Eigen's slerp and normalisation); on x86-64 they
    agree bit for bit.  The 2-ulp margin is for a host compiler that contracts a * b + c into one fused multiply-add (aarch64 gcc
    does by default): that rounds once instead of twice and can move the last bit of each product sum."""
    rng = np.random.default_rng(100 * seed + keyframe_count)
    n = 30
    frames, idx, original, current = trajectory(rng, n, keyframe_count)
    end = n - 2   # the last frame stays out of range
    ours = product(idx, original, current, start, end, frames)
    theirs = oracle(idx, original, current, start, end, frames)
    assert within_ulps(ours, theirs, 2)
    moved = [f for f in range(n) if not np.array_equal(ours[f], frames[f])]
    assert set(moved) == set(range(start, end + 1)) - set(idx.tolist())
    assert min(moved) < idx[0]
    assert max(moved) > idx[-1]
    if keyframe_count > 1:
        assert any(idx[0] < f < idx[-1] for f in moved)


@pytest.mark.parametrize("impl", ["product", "oracle"])
def test_keyframe_rows_and_rows_out_of_range_are_never_written(impl):
    rng = np.random.default_rng(3)
    frames, idx, original, current = trajectory(rng, 24, 4)
    sentinel = np.frombuffer(np.uint32(0x7fc0dead).tobytes() * 7, np.float32)   # a NaN pattern no arithmetic produces
    for i in list(idx) + [0, 1, 23]:
        frames[i] = sentinel
    out = IMPLS[impl](idx, original, current, 2, 22, frames)
    for i in list(idx) + [0, 1, 23]:
        assert out[i].tobytes() == sentinel.tobytes(), i
    assert np.isfinite(out[2:23][~np.isin(np.arange(2, 23), idx)]).all()


@pytest.mark.parametrize("impl", ["product", "oracle"])
def test_unchanged_keyframes_leave_every_frame_unchanged(impl):
    """After a BA call that moved nothing, every frame keeps its pose to fp32 rounding (a few SE3 products of poses with
    translations up to 2 m: 2e-6)."""
    rng = np.random.default_rng(4)
    frames, idx, original, _ = trajectory(rng, 30, 6)
    current = frames[idx].copy()
    out = IMPLS[impl](idx, original, current, 0, 29, frames)
    for f in range(30):
        assert same_pose(out[f], frames[f], 2e-6), f


@pytest.mark.parametrize("impl", ["product", "oracle"])
def test_one_rigid_motion_of_all_keyframes_moves_every_frame_with_them(impl):
    """G * keyframe for every keyframe: every frame becomes G * frame (the whole trajectory moved rigidly; 1e-5 for the fp32
    products of poses with translations up to 3 m)."""
    rng = np.random.default_rng(5)
    frames, idx, original, _ = trajectory(rng, 30, 6)
    G = random_pose(rng, 0.8, 1.0)
    current = np.stack([O.se3_mul(G, frames[i]) for i in idx])
    out = IMPLS[impl](idx, original, current, 0, 29, frames)
    for f in sorted(set(range(30)) - set(idx.tolist())):   # (keyframe rows are the caller's: they are not written)
        assert same_pose(out[f], O.se3_mul(G, frames[f]), 1e-5), f


@pytest.mark.parametrize("impl", ["product", "oracle"])
def test_interpolation_tends_to_the_one_sided_extrapolations(impl):
    """Keyframes at frames 0 and N: frame 1 (factor 1/N) lies within 1/N of the way from keyframe 0's extrapolation to keyframe
    N's, frame N - 1 within 1/N of keyframe N's."""
    rng = np.random.default_rng(6)
    N = 4096
    frames = np.tile(IDENT, (N + 1, 1))
    frames[1], frames[N - 1] = random_pose(rng), random_pose(rng)
    idx = np.array([0, N], np.int32)
    kf = [random_pose(rng), random_pose(rng)]
    original = np.stack([O.se3_inverse(p) for p in kf])
    current = np.stack([O.se3_mul(random_pose(rng, 0.1, 0.1), p) for p in kf])
    for f, near in ((1, 0), (N - 1, 1)):
        out = IMPLS[impl](idx, original, current, f, f, frames[:f + 1])
        near_only = T.extrapolate(original[near], current[near], frames[f])
        far_only = T.extrapolate(original[1 - near], current[1 - near], frames[f])
        gap = np.abs(near_only.astype(np.float64) - far_only).max()
        assert gap > 1e-2
        assert same_pose(out[f], near_only, 1.5 * gap / N + 2e-6), f
        assert not same_pose(out[f], near_only, 0.2 * gap / N), f   # ... and it is an interpolation, not the extrapolation


def test_interpolated_correction_at_factor_0_and_1_is_the_one_sided_correction():
    rng = np.random.default_rng(7)
    a, b = random_pose(rng, 0.3, 1.0), random_pose(rng, 0.3, 1.0)
    assert within_ulps(T.interpolate_correction(a, b, 0.0), a, 1)
    assert within_ulps(T.interpolate_correction(a, b, 1.0), b, 1)


def geodesic_slerp(q0, t, q1):
    """float64 reference: q0 * (q0^-1 q1)^t along the short arc."""
    q0, q1 = np.asarray(q0, np.float64), np.asarray(q1, np.float64)
    if np.dot(q0, q1) < 0:
        q1 = -q1
    omega = np.arccos(np.clip(np.dot(q0, q1), -1, 1))
    if omega < 1e-12:
        return q0
    return (np.sin((1 - t) * omega) * q0 + np.sin(t * omega) * q1) / np.sin(omega)


def test_slerp_branches():
    """Eigen's slerp: sin weights below |d| = 1 - eps, linear weights at and above it, and the short arc for d < 0."""
    rng = np.random.default_rng(8)
    for _ in range(50):
        q0, q1 = random_pose(rng, 1.0)[:4], random_pose(rng, 1.0)[:4]
        t = np.float32(rng.uniform(0, 1))
        assert abs(T.dot4(q0, q1)) < 1 - T.EPS_F
        assert np.abs(T.slerp(q0, t, q1) - geodesic_slerp(q0, t, q1)).max() < 1e-6
        # the opposite sign of the same rotation: the short arc, i.e. the same rotation as before up to the sign
        assert same_pose(np.concatenate([T.slerp(q0, t, -q1), [0, 0, 0]]), np.concatenate([T.slerp(q0, t, q1), [0, 0, 0]]), 1e-6)
    # |d| >= 1 - eps: linear weights, exactly (1 - t) q0 + t q1 -- and with q1 = -q0, (1 - t) q0 + t q0 = q0, not (1 - 2t) q0
    q0 = random_pose(rng, 1.0)[:4]
    q1 = q0.copy()
    q1[3] = np.nextafter(q1[3], np.float32(2))   # one ulp away: |d| rounds to the threshold or above
    assert abs(T.dot4(q0, q1)) >= 1 - T.EPS_F
    t = np.float32(0.375)
    assert np.array_equal(T.slerp(q0, t, q1), (np.float32(1) - t) * q0 + t * q1)
    assert np.array_equal(T.slerp(q0, np.float32(0.5), -q0), q0)


@pytest.mark.parametrize("impl", ["product", "oracle"])
@pytest.mark.parametrize("same_correction", [True, False], ids=["linear_branch", "sin_branch"])
def test_opposite_quaternion_sign_of_a_keyframe_takes_the_short_arc(impl, same_correction):
    """The next keyframe's pose given with -q (the same rotation): its correction's quaternion comes out negated, d < 0, and the
    interpolated frame must be the one computed with +q.  Without the sign flip of Eigen's slerp the linear branch would
    interpolate through the zero quaternion at factor 0.5."""
    rng = np.random.default_rng(9)
    frames = np.stack([random_pose(rng) for _ in range(3)])
    idx = np.array([0, 2], np.int32)
    original = np.stack([O.se3_inverse(frames[0]), O.se3_inverse(frames[2])])
    move = random_pose(rng, 0.1, 0.1)
    if same_correction:   # both keyframes moved by the same global motion: equal corrections, |d| = 1
        current = np.stack([O.se3_mul(move, frames[0]), O.se3_mul(move, frames[2])])
    else:
        current = np.stack([O.se3_mul(move, frames[0]), O.se3_mul(random_pose(rng, 0.1, 0.1), frames[2])])
    flipped = current.copy()
    flipped[1, :4] = -flipped[1, :4]
    plus = IMPLS[impl](idx, original, current, 1, 1, frames[:2])
    minus = IMPLS[impl](idx, original, flipped, 1, 1, frames[:2])
    c_prev = T.correction(original[0], flipped[0], frames[1])
    c_next = T.correction(original[1], flipped[1], frames[1])
    assert T.dot4(c_prev[:4], c_next[:4]) < 0
    assert np.isfinite(minus[1]).all()
    assert same_pose(minus[1], plus[1], 2e-6)
    if same_correction:
        assert same_pose(minus[1], O.se3_mul(move, frames[1]), 1e-5)


def test_invalid_arguments_write_nothing():
    lib = _lib.load()
    rng = np.random.default_rng(10)
    frames, idx, original, current = trajectory(rng, 12, 3)
    out = frames.copy()

    def call(K=3, i=idx, o=original, c=current, start=0, end=11, f=out):
        ptr = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data
        i = None if i is None else np.ascontiguousarray(i, np.int32)
        return lib.bba_host_deform_trajectory(K, ptr(i), ptr(o), ptr(c), start, end, ptr(f))

    bad = [dict(K=0), dict(K=-1), dict(i=np.array([4, 4, 7])), dict(i=np.array([5, 4, 7])), dict(i=np.array([-1, 4, 7])),
           dict(start=-1), dict(start=6, end=5), dict(i=None), dict(o=None), dict(c=None), dict(f=None)]
    for kw in bad:
        assert call(**kw) == _lib.ERR_INVALID_ARGUMENT, kw
        assert out.tobytes() == frames.tobytes(), kw
    assert call() == _lib.OK
    assert not np.array_equal(out, frames)
    # the Python mirror raises, clamps end_frame to the last frame like the reference, and wants an array it can update in place
    with pytest.raises(_lib.BadBAError):
        deform_trajectory(0, 11, [], original[:0], current[:0], frames.copy())
    clamped = frames.copy()
    deform_trajectory(0, 1000, idx, original, current, clamped)
    assert np.array_equal(clamped, out)
    with pytest.raises(_lib.BadBAError):
        deform_trajectory(0, 11, idx, original, current, frames.astype(np.float64))


def test_cpp_adaptor_deforms_a_video(tmp_path):
    """include/badba_direct_ba.hpp: ExtrapolateAndInterpolateKeyframePoseChanges on a libvis-shaped video (depth and colour frames
    with global_T_frame() / SetGlobalTFrame()), both frames set, keyframes and frames past the video untouched; the DirectBA
    overload and RememberKeyframePoses are instantiated (running them needs a device)."""
    gxx = shutil.which("g++")
    if gxx is None or not os.path.isdir("/usr/local/cuda/include"):
        pytest.skip("no host compiler / CUDA headers")
    rng = np.random.default_rng(11)
    frames, idx, original, current = trajectory(rng, 16, 3)
    (tmp_path / "in.bin").write_bytes(np.concatenate([frames.ravel(), original.ravel(), current.ravel()]).astype(np.float32).tobytes())
    src = tmp_path / "deform.cpp"
    src.write_text(r'''
#include <cstdio>
#include <memory>
#include "badba_direct_ba.hpp"
struct SE3f { float v[7] = {0, 0, 0, 1, 0, 0, 0}; float* data() { return v; } const float* data() const { return v; } };
struct Cam { int w, h; float p[4]; int width() const { return w; } int height() const { return h; } const float* parameters() const { return p; } };
struct Frame {
  SE3f pose; int sets = 0;
  const SE3f& global_T_frame() const { return pose; }
  void SetGlobalTFrame(const SE3f& p) { pose = p; ++sets; }
};
struct Video {
  std::vector<std::shared_ptr<Frame>> depth, color;
  size_t frame_count() const { return depth.size(); }
  std::shared_ptr<Frame>& depth_frame_mutable(int i) { return depth[i]; }
  std::shared_ptr<Frame>& color_frame_mutable(int i) { return color[i]; }
};
int main(int argc, char** argv) {
  const int n = 16, K = 3;
  std::vector<float> in(7 * (n + 2 * K));
  FILE* f = std::fopen(argv[1], "rb");
  if (!f || std::fread(in.data(), sizeof(float), in.size(), f) != in.size()) return 1;
  std::fclose(f);
  Video video;
  for (int i = 0; i < n; ++i) {
    video.depth.push_back(std::make_shared<Frame>());
    video.color.push_back(std::make_shared<Frame>());
    std::memcpy(video.depth[i]->pose.v, &in[7 * i], 28);
  }
  std::vector<SE3f> original(K), current(K);
  for (int k = 0; k < K; ++k) {
    std::memcpy(original[k].v, &in[7 * (n + k)], 28);
    std::memcpy(current[k].v, &in[7 * (n + K + k)], 28);
  }
  std::vector<int> index = {std::atoi(argv[2]), std::atoi(argv[3]), std::atoi(argv[4])};
  badba::ExtrapolateAndInterpolateKeyframePoseChanges(1u, 1000u, index, original, current, &video);   // end clamped to n - 1
  for (int i = 0; i < n; ++i) {
    const bool keyframe = i == index[0] || i == index[1] || i == index[2];
    const int expected_sets = (i == 0 || keyframe) ? 0 : 1;
    if (video.depth[i]->sets != expected_sets || video.color[i]->sets != expected_sets) return 2;
    if (expected_sets && std::memcmp(video.depth[i]->pose.v, video.color[i]->pose.v, 28) != 0) return 3;
    std::fwrite(video.depth[i]->pose.v, sizeof(float), 7, stdout);
  }
  if (argc > 100) {   // never taken: instantiates the DirectBA forms
    Cam c{64, 48, {30, 30, 32, 24}};
    badba::DirectBA<SE3f, Cam> ba(1000, 1e-3f, 40.f, 4, 0.8f, 1, 2, 3, c, c, 0, true, true);
    ba.AddKeyframe(nullptr, 7, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, {nullptr, 0}, SE3f(), 0.5f, 2.f);
    std::vector<SE3f> remembered;
    badba::RememberKeyframePoses(ba, &remembered);
    badba::ExtrapolateAndInterpolateKeyframePoseChanges(0u, 10u, ba, remembered, &video);
    return ba.keyframe_frame_index(0);
  }
  return 0;
}''')
    exe = tmp_path / "deform"
    libdir = os.path.join(ROOT, "badslam_b200")
    subprocess.check_call([gxx, "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src), "-o",
                           str(exe), "-L", libdir, "-lbadba_b200", f"-Wl,-rpath,{libdir}"])
    run = subprocess.run([str(exe), str(tmp_path / "in.bin")] + [str(i) for i in idx], capture_output=True)
    assert run.returncode == 0, run.returncode
    got = np.frombuffer(run.stdout, np.float32).reshape(16, 7)
    assert np.array_equal(got, product(idx, original, current, 1, 15, frames))
    assert within_ulps(got, oracle(idx, original, current, 1, 15, frames), 2)
