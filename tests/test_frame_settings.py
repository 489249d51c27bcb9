"""The LiDAR-to-base extrinsic and PCL >= 1.10's transform order through every path merged after the first remove / revert / ND / PD passes:
the adaptive and ball passes, scan-side removal, ICP with the refined kNN diff, the kept scan images, the orchestrator's features, the
delta maps and the driver's --pcl110.  Four frame settings: F0 (identity, order 0; the control), F1 (extrinsic, order 0), F2 (identity,
order 1) and F3 (extrinsic, order 1).

Each path picks its frames in its own code (DESIGN.md §5.1): the kNN diff and ICP move scans to the world with base2lidar, scan-side
removal and the merge with lidar2base, every path moves points back with base2lidar, and the ball is centred on the pose (the base), not on
the LiDAR.  The CPU self-checks prove that on these scenes the order changes coordinates and decisions, and that every plausible wrong
frame choice gives a different answer; the GPU tests then hold the device to the restatements bit for bit under F1, F2 and F3."""
import functools
import os
import subprocess

import numpy as np
import pytest

import oracle
import synth
import lt_mapper_b200 as ltr
from lt_mapper_b200 import removert
import _adaptive_oracle as A
import _ball_oracle as B
import _delta_oracle as D
import _icp_oracle as io
import _scanside_oracle as so
from test_gpu_project_seam import _scan_set, seam_scene

F32 = np.float32
I4 = np.eye(4)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "lt_mapper_b200", "ltremovert_b200")
FAST = {0: dict(fast_path=False), 1: dict(fast_path=True, cull=False), 2: dict(fast_path=True, cull=True)}
# (device mode, oracle mode, alpha): HD remove, revert at 0.95 r, ND and PD filter passes
VARIANTS = {"HD": (ltr.MODE_HD, oracle.MODE_HD, 2.5), "revert": (ltr.MODE_HD, oracle.MODE_HD, F32(0.95 * F32(2.5))),
            "ND": (ltr.MODE_ND, oracle.MODE_ND, 2.5), "PD": (ltr.MODE_PD, oracle.MODE_PD, 2.5)}
CRITERIA = {"map": so.MAP, "scan_minus_map": so.SCAN_MINUS_MAP}


def _rot(axis, a):
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(4)
    R[i, i] = c; R[j, j] = c; R[i, j] = -s; R[j, i] = s
    return R


# A LiDAR mounted 2.4 m above the base and 1.5 m off its centre, turned about all three axes by angles whose sines and cosines are not
# exact in binary; base2lidar is its double inverse as the orchestrator computes it (removerter.cpp's invert4x4).
L2B = _rot(2, 0.29) @ _rot(1, -0.13) @ _rot(0, 0.07)
L2B[:3, 3] = [1.35, -0.6, 2.4]
B2L = removert.inverse_poses(L2B[None])[0]
FRAMES = {"F0": (False, 0), "F1": (True, 0), "F2": (False, 1), "F3": (True, 1)}
SETTINGS = ["F1", "F2", "F3"]


class Frame:
    def __init__(self, name):
        self.name = name
        self.ext, self.order = FRAMES[name]
        self.l2b = L2B if self.ext else I4
        self.b2l = B2L if self.ext else I4

    def ctx(self, **kw):
        return ltr.Context(lidar2base=self.l2b, base2lidar=self.b2l, transform_order=self.order, **kw)

    def flipped(self):
        """the same extrinsic with the other transform order"""
        return Frame({(False, 0): "F2", (True, 0): "F3", (False, 1): "F0", (True, 1): "F1"}[(self.ext, self.order)])


def _same(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _bits_share(a, b):
    """share of the points whose xyz bits differ between a and b (same shape)"""
    a, b = np.ascontiguousarray(a[:, :3], F32), np.ascontiguousarray(b[:, :3], F32)
    return float((a.view(np.uint32) != b.view(np.uint32)).any(1).mean())


def _per_kf(pts, off):
    return [pts[off[j]:off[j + 1]] for j in range(len(off) - 1)]


# ---------------------------------------------------------------------------------------------------------------------------- scenes
N_PLANE = 300


def scene_session(s, ext, seed=0):
    """The session as the LiDAR (mounted by L2B when ext) records it, with a wall added on the world plane x = 0.

    Each scan is re-expressed in the LiDAR frame and the base poses are kept, so the world stays where it was (pose @ L2B @ scan = pose @
    scan up to f32 rounding) and both sessions and all keyframes still agree on the map.  The two transform orders differ by a few double
    ulps of the partial sums, which no f32 result shows where the result is as large as the terms; at the wall, global x is ~1e-6 while
    the terms are ~60 m, so the order changes the bits of several per cent of the wall's points (the last N_PLANE of every scan).  The
    N_PLANE points before them lie straight ahead of the LiDAR (local y = 0), where the way back to the LiDAR frame shows the order, and
    the N_PLANE before those are the wall again as the kNN diff and ICP see it (base2lidar, then the pose)."""
    rng = np.random.default_rng(seed)
    scans = []
    for k in range(s.K):
        P = s.poses[k]
        g = np.zeros((N_PLANE, 4), F32)
        g[:, 1] = P[1, 3] + rng.uniform(-20.0, 20.0, N_PLANE)
        g[:, 2] = P[2, 3] + rng.uniform(-2.0, 6.0, N_PLANE)
        wall = so.global2local(g, oracle.inverse4x4(P), B2L if ext else I4)
        kwall = so.global2local(g[::-1], oracle.inverse4x4(P), L2B if ext else I4)   # the same wall for the kNN diff's base2lidar
        ahead = np.zeros((N_PLANE, 4), F32)   # local y = 0: moved to the world and back, y is ~1e-6 and the order shows again
        ahead[:, 0] = rng.uniform(5.0, 40.0, N_PLANE)
        ahead[:, 2] = rng.uniform(-3.0, 3.0, N_PLANE)
        scans.append(np.concatenate([oracle.transform(s.scan(k), B2L) if ext else s.scan(k), kwall, ahead, wall]))
    xyzi, off = _scan_set(scans)
    return synth.SessionData(xyzi, off, s.poses.copy())


def lidar_session(s):
    return scene_session(s, True)


def wall(s, fr):
    """the wall points of every keyframe, in the world, under frame setting fr (local2global)"""
    return np.concatenate([so.local2global(s.scan(k)[-N_PLANE:], s.poses[k], fr.l2b, fr.order) for k in range(s.K)])


TINY = 1e-30   # a kNN threshold below every non-zero squared distance of these scenes


def exact_map(m, s, fr):
    """the map plus the wall's global points of session s under fr, bit for bit"""
    return np.concatenate([m, wall(s, fr)])


def kwall(s, fr, order=None):
    """the kNN diff's wall points of every keyframe, in the world as ltr_knn_diff moves them (base2lidar, then the pose)"""
    o = fr.order if order is None else order
    return [io.global_scan(s.scan(k)[-3 * N_PLANE:-2 * N_PLANE], s.poses[k], fr.b2l, o) for k in range(s.K)]


# ------------------------------------------------------------------------------------------------------------------- order scene
ORDER_POSE = _rot(2, 0.31) @ _rot(1, 0.05) @ _rot(0, -0.04)
ORDER_POSE[:3, 3] = [12.0, 3.0, 0.5]
SEAM_RETURN_AZ = np.deg2rad(179.6)   # inside the last column at every resolution the tests use, clear of its edges


def flip_points(M, n, rng, span=400):
    """n f32 points p with (M p).x < -5 m, elevation within 20 degrees, whose (M p).y has one sign bit under transform order 0 and the
    other under order 1.  Such a point lies on the plane local y = 0 near a plane p_j = 0 of the input frame: the other two coordinates
    put it within ~1e-6 of local y = 0, and p_j, tiny and so with ulps of ~1e-13, is walked until the two orders' double partial sums,
    which differ by a few ulps of terms of metres, round to opposite signs.  On the azimuth seam atan2 turns that sign into the first or
    the last column of the range image."""
    M = np.asarray(M, np.float64)
    out = []
    for _ in range(20000):
        if len(out) >= n:
            break
        j = int(rng.integers(3))
        a, b = [i for i in range(3) if i != j]
        pa = F32(rng.uniform(-40.0, 40.0))
        pb = F32(-(M[1, a] * np.float64(pa) + M[1, 3]) / M[1, b])
        pj = F32(-(M[1, a] * np.float64(pa) + M[1, b] * np.float64(pb) + M[1, 3]) / M[1, j])
        vals, lo, hi = [pj], pj, pj
        for _ in range(span):
            lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
            vals += [lo, hi]
        cand = np.zeros((len(vals), 4), F32)
        cand[:, j] = vals; cand[:, a] = pa; cand[:, b] = pb
        l0, l1 = oracle.transform(cand, M, 0), oracle.transform(cand, M, 1)
        el = np.degrees(np.arctan2(l0[:, 2], -l0[:, 0]))
        ok = (np.signbit(l0[:, 1]) != np.signbit(l1[:, 1])) & (l0[:, 0] < -5) & (l1[:, 0] < -5) & (np.abs(el) < 20)
        ok &= np.linalg.norm(l0[:, :3], axis=1) < 60
        if ok.any():
            out.append(cand[np.flatnonzero(ok)[0]])
    assert len(out) == n, len(out)
    return np.array(out)


@functools.lru_cache(maxsize=None)
def _order_scene(name, nd):
    return order_scene(Frame(name), nd)


def order_scene(fr, nd=False, n=16, seed=5):
    """One keyframe whose map points sit on the azimuth seam behind the LiDAR, each at the sign of local y that the transform order
    picks (flip_points), with a scan return at the point's elevation in the last seam column only, 2 m behind the point (HD / PD) or in
    front of it (nd).  The point whose order puts it in the last column is flagged, the other one finds no return.  With the extrinsic
    the pose is the identity (exact in both orders) and base2lidar carries the order; without it the pose does.
    Returns (map, scan xyzi, offsets, poses, inverse poses)."""
    rng = np.random.default_rng(seed)
    pose = I4 if fr.ext else ORDER_POSE
    inv = oracle.inverse4x4(pose)
    p = flip_points(B2L if fr.ext else inv, n, rng)
    local = so.global2local(p, inv, fr.b2l, fr.order).astype(np.float64)
    r = np.linalg.norm(local[:, :3], axis=1)
    el = np.arctan2(local[:, 2], np.hypot(local[:, 0], local[:, 1]))
    s = r + (-2.0 if nd else 2.0)
    scan = np.stack([s * np.cos(el) * np.cos(SEAM_RETURN_AZ), s * np.cos(el) * np.sin(SEAM_RETURN_AZ), s * np.sin(el), np.zeros(n)], 1)
    m = p.copy()
    m[:, 3] = 1.0
    return m, scan.astype(F32), np.array([0, n], np.int64), pose[None], inv[None]


def global_map(s, fr, leaf=0.05):
    """makeGlobalMap of a session under frame setting fr: lidar2base, then the pose, in fr's order, voxelised"""
    return D.merged_map([s.scan(k) for k in range(s.K)], s.poses, leaf, fr.l2b, fr.order)


@pytest.fixture(scope="module")
def scenes(small_pair):
    """per extrinsic flag: (central, query) sessions, and per frame setting: the two sessions' global maps"""
    sess = {ext: tuple(scene_session(s, ext, j) for j, s in enumerate(small_pair)) for ext in (False, True)}
    maps = {n: [global_map(s, Frame(n)) for s in sess[FRAMES[n][0]]] for n in FRAMES}
    return sess, maps


def _map_for(maps, name, mode):
    return maps[name][0] if mode == ltr.MODE_HD else maps[name][1][::7]   # the filter passes project the other session's map


def _radius(m, poses):
    """a radius at which every keyframe's ball holds between 10 and 90 % of the map"""
    d = np.stack([np.sqrt(B.sq_dist(m, c).astype(np.float64)) for c in B.centres(poses)])
    lo, hi = np.quantile(d, 0.1, axis=1).max(), np.quantile(d, 0.9, axis=1).min()
    assert lo < hi, (lo, hi)
    return float(F32(lo + 0.3 * (hi - lo)))


def seam_scene_in(fr, seed=4, K=8):
    """test_gpu_project_seam's seam scene with the LiDAR where the scene's sensor was: the base poses are pose @ base2lidar."""
    m, scans, poses, _, _ = seam_scene(seed, K, 50.0, nonrigid=(5,), nonfinite=True)
    if fr.ext:
        poses = np.stack([p @ B2L for p in poses])
    return m, scans, poses, oracle.inverse_poses(poses)


def _shell(rng, c, r2, n):
    """points whose d2 from c is r2 (outside), one ulp below (inside) or one ulp above: ulp walks of points on the sphere"""
    out = []
    R = np.sqrt(np.float64(r2))
    want = {F32(r2), np.nextafter(F32(r2), F32(0)), np.nextafter(F32(r2), F32(np.inf))}
    while len(out) < n:
        v = rng.normal(size=3)
        v[2] *= 0.1
        p = (c.astype(np.float64) + R * v / np.linalg.norm(v)).astype(F32)
        for _ in range(64):
            d2 = B.sq_dist(p[None], c)[0]
            if d2 in want:
                out.append(p.copy())
                break
            j = rng.integers(3)
            p[j] = np.nextafter(p[j], F32(np.inf) if (d2 < r2) == (p[j] < c[j]) else F32(-np.inf))
    return np.array(out, F32)


def boundary_map(c, base_map, radius, n=300, k_shells=4, seed=11):
    """the map plus, for each of the first k_shells keyframes, points on the sphere of `radius` around its pose centre, to the ulp"""
    rng = np.random.default_rng(seed)
    r2 = B.radius2(radius)
    cs = B.centres(c.poses)
    pts = np.concatenate([_shell(rng, cc, r2, n) for cc in cs[:k_shells]])
    return np.concatenate([base_map, np.concatenate([pts, np.zeros((len(pts), 1), F32)], 1)])


def _perturb(poses, trans=0.3, deg=1.0):
    E = _rot(2, np.deg2rad(deg)) @ _rot(0, np.deg2rad(deg / 3))
    E[:3, 3] = np.array([1.0, -0.6, 0.2]) * trans
    return np.stack([p @ E for p in poses])


def icp_target(q, fr):
    """the other session's map in the frame ltr_knn_diff moves scans to (base2lidar, then the pose), so that keyframes register"""
    g = np.concatenate([io.global_scan(q.scan(k), q.poses[k], fr.b2l, fr.order) for k in range(q.K)])
    m = oracle.voxel(g, 0.05)
    return m, oracle.voxel(m, 0.4)


# ======================================================================================================== 1. frame matrix (CPU)
def test_extrinsic_is_the_one_the_issue_needs():
    assert np.array_equal(B2L, oracle.inverse4x4(L2B)), "base2lidar must be the double inverse both restatements use"
    R = L2B[:3, :3]
    assert all(abs(R[i, j]) > 0.05 for i in range(3) for j in range(3) if i != j), "a rotation about every axis"
    assert L2B[2, 3] >= 2.0 and np.linalg.norm(L2B[:3, 3]) > 2.5
    assert not np.array_equal(B2L @ L2B, I4) and np.abs(B2L @ L2B - I4).max() < 1e-14
    assert not np.array_equal(B2L, L2B.T)   # lidar2base and base2lidar are not interchangeable


# ============================================================================================ 2. non-vacuity self-checks (CPU)
@pytest.mark.parametrize("ext", [False, True])
def test_order_changes_the_transformed_points(scenes, ext):
    sess, _ = scenes
    c = sess[ext][0]
    fr = Frame("F1" if ext else "F0")
    g = {0: wall(c, fr), 1: wall(c, fr.flipped())}
    share = _bits_share(g[0], g[1])
    rest = np.concatenate([so.local2global(c.scan(k)[:-N_PLANE], c.poses[k], fr.l2b, 0) for k in range(c.K)])
    rest1 = np.concatenate([so.local2global(c.scan(k)[:-N_PLANE], c.poses[k], fr.l2b, 1) for k in range(c.K)])
    print(f"extrinsic {ext}: the order changes {share:.3f} of the wall's global points, {_bits_share(rest, rest1):.2e} of the others")
    assert share > 0.03
    ahead = {o: np.concatenate([so.global2local(so.local2global(c.scan(k)[-2 * N_PLANE:-N_PLANE], c.poses[k], fr.l2b, 0),
                                                oracle.inverse4x4(c.poses[k]), fr.b2l, o) for k in range(c.K)]) for o in (0, 1)}
    print(f"extrinsic {ext}: the order changes {_bits_share(ahead[0], ahead[1]):.3f} of the points ahead on their way back")
    assert _bits_share(ahead[0], ahead[1]) > (0.005 if ext else 0.03)   # with the extrinsic the last step's terms are metres, not tens


@pytest.mark.parametrize("name", SETTINGS)
def test_adaptive_settings_matter(scenes, name):
    fr = Frame(name)
    sess, maps = scenes
    c = sess[fr.ext][0]
    inv = oracle.inverse_poses(c.poses)
    for variant in ("HD", "ND"):
        _, omode, alpha = VARIANTS[variant]
        m = _map_for(maps, name, VARIANTS[variant][0])
        right = A.remove_pass(m, c.xyzi, c.offsets, inv, omode, alpha, 0.05, lidar2base=fr.l2b, order=fr.order)
        assert right.sum() > 0
        wrong = {}
        if fr.ext:
            wrong["no extrinsic"] = A.remove_pass(m, c.xyzi, c.offsets, inv, omode, alpha, 0.05, order=fr.order)
            wrong["lidar2base for base2lidar"] = A.remove_pass(m, c.xyzi, c.offsets, inv, omode, alpha, 0.05, lidar2base=B2L, order=fr.order)
        for why, w in wrong.items():
            assert not np.array_equal(w, right), (variant, why)
    if fr.ext:   # test_adaptive_seam_scene's scene
        m, scans, poses, inv = seam_scene_in(fr)
        xyzi, off = _scan_set(scans)
        fin = np.isfinite(m[:, :3]).all(1)
        for omode in (oracle.MODE_HD, oracle.MODE_PD, oracle.MODE_ND):
            right = A.remove_pass(m[fin], xyzi, off, inv, omode, 2.5, 0.05, lidar2base=fr.l2b, order=fr.order)
            assert right.sum() > 0
            for why, l2b in (("no extrinsic", I4), ("lidar2base for base2lidar", B2L)):
                assert not np.array_equal(A.remove_pass(m[fin], xyzi, off, inv, omode, 2.5, 0.05, lidar2base=l2b, order=fr.order), right), why


def _order_scene_flags(name, nd, mode, alpha, kind, order=None, l2b=None):
    fr = Frame(name)
    m, scan, off, poses, inv = _order_scene(name, nd)
    o = fr.order if order is None else order
    l2b = fr.l2b if l2b is None else l2b
    if kind == "const":
        return oracle.remove_pass(m, scan, off, inv, mode, alpha, lidar2base=l2b, order=o)
    if kind == "adaptive":
        return A.remove_pass(m, scan, off, inv, mode, alpha, 0.05, lidar2base=l2b, order=o)
    return B.remove_pass(m, scan, off, poses, inv, mode, alpha, ORDER_BALL, 0.1, 0.05, lidar2base=l2b, order=o)


ORDER_BALL = 100.0
ORDER_CASES = [(nd, mode, alpha) for nd, modes in ((False, (oracle.MODE_HD, oracle.MODE_PD)), (True, (oracle.MODE_ND,)))
               for mode in modes for alpha in (2.5, 1.0)]


@pytest.mark.parametrize("name", SETTINGS)
def test_order_scene_makes_the_order_decide(name):
    """the constant, adaptive and ball passes on the order scene: the other order, no extrinsic and lidar2base for base2lidar each change
    flags, for every mode and both resolutions the device test runs"""
    fr = Frame(name)
    for nd, mode, alpha in ORDER_CASES:
        for kind in ("const", "adaptive", "ball"):
            right = _order_scene_flags(name, nd, mode, alpha, kind)
            wrong = {"order": _order_scene_flags(name, nd, mode, alpha, kind, order=1 - fr.order)}
            if fr.ext:
                wrong["no extrinsic"] = _order_scene_flags(name, nd, mode, alpha, kind, l2b=I4)
                wrong["lidar2base for base2lidar"] = _order_scene_flags(name, nd, mode, alpha, kind, l2b=B2L)
            for why, w in wrong.items():
                assert not np.array_equal(w, right), (nd, mode, alpha, kind, why)


@pytest.mark.parametrize("name", SETTINGS)
def test_ball_settings_matter(scenes, name):
    fr = Frame(name)
    sess, maps = scenes
    c = sess[fr.ext][0]
    inv = oracle.inverse_poses(c.poses)
    m = maps[name][0]
    radius = _radius(m, c.poses)
    for thres, coeff in ((0.1, 0.0), (0.1, 0.05)):
        def run(poses=c.poses, l2b=fr.l2b, order=fr.order, mm=m):
            return B.remove_pass(mm, c.xyzi, c.offsets, poses, inv, oracle.MODE_HD, 2.5, radius, thres, coeff, lidar2base=l2b, order=order)
        right = run()
        assert right.sum() > 0
        wrong = {}
        if fr.ext:
            wrong["no extrinsic"] = run(l2b=I4)
            wrong["lidar2base for base2lidar"] = run(l2b=B2L)
            # the ball around the LiDAR: same projection, centres at the translation of pose @ lidar2base
            wrong["ball at the LiDAR"] = run(poses=np.stack([p @ L2B for p in c.poses]))
        for why, w in wrong.items():
            assert not np.array_equal(w, right), (coeff, why)
        if fr.ext:
            # test_ball_boundary_scene's scene: its shell points decide differently around the base and around the LiDAR
            r9 = F32(9.0)
            mb = boundary_map(c, m, r9)
            at_base = B.remove_pass(mb, c.xyzi, c.offsets, c.poses, inv, oracle.MODE_HD, 2.5, r9, thres, coeff, lidar2base=fr.l2b,
                                    order=fr.order)
            at_lidar = B.remove_pass(mb, c.xyzi, c.offsets, np.stack([p @ L2B for p in c.poses]), inv, oracle.MODE_HD, 2.5, r9, thres, coeff,
                                     lidar2base=fr.l2b, order=fr.order)
            assert not np.array_equal(at_base[len(m):], at_lidar[len(m):]), coeff


@pytest.mark.parametrize("name", SETTINGS)
def test_scanside_settings_matter(scenes, name):
    fr = Frame(name)
    sess, maps = scenes
    c = sess[fr.ext][0].subset(0, 2)
    m = maps[name][0]
    for crit in (so.MAP, so.SCAN_MINUS_MAP):
        def masks(l2b, b2l, order):
            return np.concatenate([so.split_scan(c.scan(k), c.poses[k], oracle.inverse4x4(c.poses[k]), m, crit, 3, 0.05, l2b, b2l, order)[2]
                                   for k in range(c.K)])
        right = masks(fr.l2b, fr.b2l, fr.order)
        assert 0 < right.sum() < len(right)
        wrong = {}
        if fr.ext:
            wrong["no extrinsic"] = masks(I4, I4, fr.order)
            wrong["base2lidar for lidar2base"] = masks(B2L, fr.b2l, fr.order)
        for why, w in wrong.items():
            assert not np.array_equal(w, right), (crit, why)
    # the order decides the split where the map holds the wall's global points bit for bit (k = 1, thr below every non-zero distance):
    # under the right order they are static, under the other one the wall points whose bits moved are dynamic
    me = exact_map(maps[name][0], c, fr)
    for crit in (so.MAP, so.SCAN_MINUS_MAP):
        def split(order):
            return [so.split_scan(c.scan(k), c.poses[k], oracle.inverse4x4(c.poses[k]), me, crit, 1, TINY, fr.l2b, fr.b2l, order)
                    for k in range(c.K)]
        right, flip = split(fr.order), split(1 - fr.order)
        assert all(r[2][-N_PLANE:].all() for r in right), crit
        assert not np.array_equal(np.concatenate([r[2] for r in right]), np.concatenate([f[2] for f in flip])), crit
        assert not all(_same(r[0], f[0]) for r, f in zip(right, flip)), crit


@pytest.mark.parametrize("name", ["F1", "F3"])
def test_icp_settings_matter(scenes, name):
    fr = Frame(name)
    sess, _ = scenes
    c, q = (s.subset(0, 2) for s in sess[fr.ext])
    poses = _perturb(c.poses)
    tgt, tgt_down = icp_target(q, fr)
    right = io.refine_session(c.xyzi, c.offsets, poses, tgt_down, fr.b2l, fr.order)
    assert (right[1] < 1.0).any(), "no keyframe registers: the acceptance test decides nothing"
    # The order moves source coordinates only where they are ~1e-6 (the wall), by ~1e-13; T is an f32 mean over thousands of points and
    # moves by no bit.  Where the order does decide in this path is the refined partition: test_refined_diff_order_decides.
    wrong = {}
    if fr.ext:
        wrong["no extrinsic"] = io.refine_session(c.xyzi, c.offsets, poses, tgt_down, I4, fr.order)
        wrong["lidar2base for base2lidar"] = io.refine_session(c.xyzi, c.offsets, poses, tgt_down, L2B, fr.order)
    for why, w in wrong.items():
        assert not _same(w[0], right[0]) and not np.array_equal(w[1], right[1]), why

def exact_knn_target(tgt, c, fr):
    """the kNN target plus the kNN diff's wall points of the scanned keyframes under fr, bit for bit"""
    return np.concatenate([tgt] + kwall(c, fr))


@pytest.mark.parametrize("name", SETTINGS)
def test_refined_diff_order_decides(scenes, name):
    """ltr_knn_diff_refined's partition against a target that holds the scanned keyframes' wall points bit for bit (k = 1, thr below every
    non-zero distance, keyframes not accepted): under the right order the wall coexists, under the other one the wall points whose bits
    moved are diff points; no extrinsic and lidar2base for base2lidar move every wall point"""
    fr = Frame(name)
    sess, _ = scenes
    c, q = (s.subset(0, 2) for s in sess[fr.ext])
    tgt = exact_knn_target(icp_target(q, fr)[0], c, fr)
    inv = oracle.inverse_poses(c.poses)
    T = np.repeat(np.eye(4, dtype=F32)[None], c.K, 0)
    acc = np.zeros(c.K, bool)

    def diff_sizes(b2l, order):
        return [len(d) for d in io.knn_diff_refined(c.xyzi, c.offsets, c.poses, inv, tgt, 1, TINY, T, acc, b2l, order)[1]]
    right = diff_sizes(fr.b2l, fr.order)
    wrong = {"order": diff_sizes(fr.b2l, 1 - fr.order)}
    if fr.ext:
        wrong["no extrinsic"] = diff_sizes(I4, fr.order)
        wrong["lidar2base for base2lidar"] = diff_sizes(L2B, fr.order)
    for why, w in wrong.items():
        assert all(a > b for a, b in zip(w, right)), (why, w, right)


@pytest.mark.parametrize("name", SETTINGS)
def test_delta_merge_settings_matter(scenes, name):
    fr = Frame(name)
    sess, _ = scenes
    c = sess[fr.ext][0]
    scans = [c.scan(k) for k in range(c.K)]
    right = D.merged_map(scans, c.poses, lidar2base=fr.l2b, order=fr.order)
    flip = D.merged_map(scans, c.poses, lidar2base=fr.l2b, order=1 - fr.order)
    assert not _same(right, flip)
    if fr.ext:
        assert not _same(right, D.merged_map(scans, c.poses, order=fr.order))
        assert not _same(right, D.merged_map(scans, c.poses, lidar2base=B2L, order=fr.order))
    # a near / far label of the delta primitive moves with the frame the scans were merged in
    t = wall(c, fr)
    assert not D.far_mask(t, t, 1, TINY).any() and D.far_mask(wall(c, fr.flipped()), t, 1, TINY).any()


# ========================================================================================= 3. device against restatement (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", SETTINGS)
def test_adaptive_pass(scenes, name, variant):
    fr = Frame(name)
    sess, maps = scenes
    c = sess[fr.ext][0]
    mode, omode, alpha = VARIANTS[variant]
    m = _map_for(maps, name, mode)
    inv = oracle.inverse_poses(c.poses)
    exp = {coeff: A.remove_pass(m, c.xyzi, c.offsets, inv, omode, alpha, coeff, lidar2base=fr.l2b, order=fr.order) for coeff in (0.05, 0.2)}
    assert all(e.sum() > 0 for e in exp.values())
    for fast in FAST:
        with fr.ctx(keyframe_batch=32, **FAST[fast]) as ctx:
            mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
            for coeff, e in exp.items():
                n = ctx.remove_pass_adaptive(mh, ss, ps, mode, alpha, coeff)
                got = ctx.flags_download(mh)
                assert n == int(e.sum()) and np.array_equal(got, e), (fast, coeff, np.flatnonzero(got != e)[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("name", SETTINGS)
def test_order_scene_passes(name):
    """the constant, adaptive and ball passes on the scene where the transform order decides flags (test_order_scene_makes_the_order_decide)"""
    fr = Frame(name)
    bad = []
    for nd, mode, alpha in ORDER_CASES:
        m, scan, off, poses, inv = _order_scene(name, nd)
        dmode = {oracle.MODE_HD: ltr.MODE_HD, oracle.MODE_PD: ltr.MODE_PD, oracle.MODE_ND: ltr.MODE_ND}[mode]
        for fast in FAST:
            with fr.ctx(**FAST[fast]) as ctx:
                mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(scan, off); ps = ctx.poses_upload(poses, inv)
                for kind in ("const", "adaptive", "ball"):
                    if kind == "const":
                        ctx.remove_pass(mh, ss, ps, dmode, alpha)
                    elif kind == "adaptive":
                        ctx.remove_pass_adaptive(mh, ss, ps, dmode, alpha, 0.05)
                    else:
                        ctx.remove_pass_ball(mh, ss, ps, dmode, alpha, ORDER_BALL, 0.1, 0.05)
                    got, exp = ctx.flags_download(mh), _order_scene_flags(name, nd, mode, alpha, kind)
                    if not np.array_equal(got, exp):
                        bad.append((nd, mode, alpha, fast, kind, np.flatnonzero(got != exp).tolist()))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("name", SETTINGS)
def test_adaptive_seam_scene(name):
    fr = Frame(name)
    m, scans, poses, inv = seam_scene_in(fr)
    xyzi, off = _scan_set(scans)
    fin = np.isfinite(m[:, :3]).all(1)
    bad = []
    for mode, omode in ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_PD, oracle.MODE_PD), (ltr.MODE_ND, oracle.MODE_ND)):
        exp = np.zeros(len(m), np.uint8)
        exp[fin] = A.remove_pass(m[fin], xyzi, off, inv, omode, 2.5, 0.05, lidar2base=fr.l2b, order=fr.order)
        assert exp.sum() > 0
        for Bk in (32, 3):
            for fast in FAST:
                with fr.ctx(keyframe_batch=Bk, **FAST[fast]) as ctx:
                    mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(xyzi, off); ps = ctx.poses_upload(poses, inv)
                    ctx.remove_pass_adaptive(mh, ss, ps, mode, 2.5, 0.05)
                    got = ctx.flags_download(mh)
                if not np.array_equal(got, exp):
                    bad.append((mode, Bk, fast, np.flatnonzero(got != exp)[:5].tolist()))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["HD", "ND", "PD"])
@pytest.mark.parametrize("name", SETTINGS)
def test_ball_pass(scenes, name, variant):
    fr = Frame(name)
    sess, maps = scenes
    c = sess[fr.ext][0]
    mode, omode, alpha = VARIANTS[variant]
    m = _map_for(maps, name, mode)
    inv = oracle.inverse_poses(c.poses)
    radius = _radius(m, c.poses)
    for thres, coeff in ((0.1, 0.0), (0.1, 0.05)):
        exp = B.remove_pass(m, c.xyzi, c.offsets, c.poses, inv, omode, alpha, radius, thres, coeff, lidar2base=fr.l2b, order=fr.order)
        assert exp.sum() > 0
        for fast in (0, 2):
            with fr.ctx(keyframe_batch=32, **FAST[fast]) as ctx:
                mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
                n = ctx.remove_pass_ball(mh, ss, ps, mode, alpha, radius, thres, coeff)
                got = ctx.flags_download(mh)
            assert n == int(exp.sum()) and np.array_equal(got, exp), (coeff, fast, np.flatnonzero(got != exp)[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("name", SETTINGS)
def test_ball_boundary_scene(scenes, name):
    """points one ulp either side of the spheres around the pose centres (several keyframes per launch)"""
    fr = Frame(name)
    sess, maps = scenes
    c = sess[fr.ext][0]
    inv = oracle.inverse_poses(c.poses)
    radius = F32(9.0)
    m = boundary_map(c, maps[name][0], radius)
    n0 = len(maps[name][0])
    for thres, coeff in ((0.1, 0.0), (0.1, 0.05)):
        exp = B.remove_pass(m, c.xyzi, c.offsets, c.poses, inv, oracle.MODE_HD, 2.5, radius, thres, coeff, lidar2base=fr.l2b, order=fr.order)
        assert exp[n0:].sum() > 0, "no shell point flagged: the scene does not test the sphere"
        for fast in (0, 2):
            with fr.ctx(keyframe_batch=32, **FAST[fast]) as ctx:
                mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
                n = ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, radius, thres, coeff)
                got = ctx.flags_download(mh)
            assert n == int(exp.sum()) and np.array_equal(got, exp), (coeff, fast, np.flatnonzero(got != exp)[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("criterion", list(CRITERIA))
@pytest.mark.parametrize("name", SETTINGS)
def test_scanside_split(scenes, name, criterion):
    fr = Frame(name)
    sess, maps = scenes
    s = sess[fr.ext][1].subset(0, 3)
    inv = oracle.inverse_poses(s.poses)
    crit = CRITERIA[criterion]
    cases = [(maps[name][0], k, thr) for k, thr in ((1, 0.01), (3, 0.1), (16, 0.5))]
    cases.append((exact_map(maps[name][0], s, fr), 1, TINY))   # the order decides the wall's points (test_scanside_settings_matter)
    with fr.ctx() as ctx:
        ss = ctx.scanset_upload(s.xyzi, s.offsets); ps = ctx.poses_upload(s.poses, inv)
        for m, k, thr in cases:
            mh = ctx.cloud_upload(m)
            st, dy = ctx.scanside_split(ss, ps, mh, crit, k, thr)
            ctx.cloud_free(mh)
            exp = so.split_session(s.xyzi, s.offsets, s.poses, inv, m, crit, k, thr, fr.l2b, fr.b2l, fr.order)
            for part, h in enumerate((st, dy)):
                got = _per_kf(*ctx.scanset_download(h))
                ctx.scanset_free(h)
                for kf in range(s.K):
                    assert _same(got[kf], exp[part][kf]), (k, part, kf)
            assert sum(map(len, exp[0])) > 0 and sum(map(len, exp[1])) > 0

def _icp_run(ctx, fr, xyzi, offsets, poses, target_down, target, k=2, thr=0.01, pose_offset=0):
    """tests/test_gpu_icp.py's _run with the frame setting: refinement + refined partition against the restatement, bit for bit"""
    inv = oracle.inverse_poses(poses)
    ss = ctx.scanset_upload(xyzi, offsets); ps = ctx.poses_upload(poses, inv)
    td = ctx.cloud_upload(target_down); th = ctx.cloud_upload(target)
    T, fit, it, ex = ctx.icp_refine(ss, ps, td, pose_offset=pose_offset)
    eT, efit, eit, eex = io.refine_session(xyzi, offsets, poses, target_down, fr.b2l, fr.order, pose_offset=pose_offset)
    assert np.array_equal(it, eit) and np.array_equal(ex, eex), (it, eit, ex, eex)
    assert _same(T, eT), np.abs(T - eT).max()
    assert np.array_equal(fit.view(np.uint64), efit.view(np.uint64)), (fit, efit)
    acc = fit < 1.0
    co, di = ctx.knn_diff_refined(ss, ps, th, k, thr, T, acc, pose_offset=pose_offset)
    exp = io.knn_diff_refined(xyzi, offsets, poses, inv, target, k, thr, eT, acc, fr.b2l, fr.order, pose_offset=pose_offset)
    for part, h in enumerate((co, di)):
        got = _per_kf(*ctx.scanset_download(h))
        ctx.scanset_free(h)
        for kf in range(len(offsets) - 1):
            assert _same(got[kf], exp[part][kf]), (part, kf)
    ctx.scanset_free(ss)
    ctx.poses_free(ps); ctx.cloud_free(td); ctx.cloud_free(th)
    return acc


@pytest.mark.gpu
@pytest.mark.parametrize("perturbed", [False, True])
@pytest.mark.parametrize("name", SETTINGS)
def test_icp_refine_and_refined_diff(scenes, name, perturbed):
    """keyframes 2..4 of the central session against the full pose table (pose_offset 2), registered to the query session's map"""
    fr = Frame(name)
    sess, _ = scenes
    full, q = sess[fr.ext]
    s = full.subset(2, 5)
    poses = _perturb(full.poses, 0.2, 0.5) if perturbed else full.poses
    tgt, tgt_down = icp_target(q, fr)
    with fr.ctx() as ctx:
        acc = _icp_run(ctx, fr, s.xyzi, s.offsets, poses, tgt_down, tgt, pose_offset=2)
        # the refined partition where the order decides (test_refined_diff_order_decides), rejected keyframes
        ss = ctx.scanset_upload(s.xyzi, s.offsets); ps = ctx.poses_upload(poses, oracle.inverse_poses(poses))
        sub = synth.SessionData(s.xyzi, s.offsets, poses[2:5])
        exact = exact_knn_target(tgt, sub, fr)
        th = ctx.cloud_upload(exact)
        T = np.repeat(np.eye(4, dtype=F32)[None], s.K, 0)
        rej = np.zeros(s.K, bool)
        co, di = ctx.knn_diff_refined(ss, ps, th, 1, TINY, T, rej, pose_offset=2)
        exp = io.knn_diff_refined(s.xyzi, s.offsets, poses, oracle.inverse_poses(poses), exact, 1, TINY, T, rej, fr.b2l, fr.order, pose_offset=2)
        for part, h in enumerate((co, di)):
            got = _per_kf(*ctx.scanset_download(h))
            assert all(_same(a, b) for a, b in zip(got, exp[part])), part
    assert acc.any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SETTINGS)
def test_kept_images_alternate_constant_adaptive_and_ball(scenes, name, monkeypatch):
    monkeypatch.delenv("LTR_SCAN_IMAGE_CACHE_MB", raising=False)
    fr = Frame(name)
    sess, maps = scenes
    c = sess[fr.ext][0]
    m = maps[name][0]
    inv = oracle.inverse_poses(c.poses)
    radius = _radius(m, c.poses)
    calls = [("const", 0.0), ("ball", 0.0), ("adaptive", 0.05), ("const", 0.0), ("ball", 0.05), ("adaptive", 0.2), ("ball", 0.0),
             ("adaptive", 0.05), ("const", 0.0)]

    def one(ctx, mh, ss, ps, kind, coeff):
        if kind == "const":
            ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)
        elif kind == "adaptive":
            ctx.remove_pass_adaptive(mh, ss, ps, ltr.MODE_HD, 2.5, coeff)
        else:
            ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, radius, 0.1, coeff)
        return ctx.flags_download(mh)

    fresh = {}
    for call in set(calls):
        with fr.ctx() as ctx:
            fresh[call] = one(ctx, ctx.cloud_upload(m), ctx.scanset_upload(c.xyzi, c.offsets), ctx.poses_upload(c.poses, inv), *call)
    assert np.array_equal(fresh[("const", 0.0)], oracle.remove_pass(m, c.xyzi, c.offsets, inv, oracle.MODE_HD, 2.5, lidar2base=fr.l2b,
                                                                    order=fr.order))
    assert len({fresh[k].tobytes() for k in fresh}) == len(fresh), "every call must give its own flags"
    with fr.ctx() as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        for call in calls:
            assert np.array_equal(one(ctx, mh, ss, ps, *call), fresh[call]), call


# ========================================================================================================== 4. orchestrator (F3)
F3 = Frame("F3")


def _orchestrator(c, q, q_poses=None, **kw):
    G = removert.Removerter(lidar2base=L2B, transform_order=1, **kw)
    qp = q.poses if q_poses is None else q_poses
    G.load_session(0, c.xyzi, c.offsets, c.poses, oracle.inverse_poses(c.poses))
    G.load_session(1, q.xyzi, q.offsets, qp, oracle.inverse_poses(qp))
    return G


@pytest.mark.gpu
def test_orchestrator_icp_refinement(scenes):
    """Step 2 with the refinement on equals ltr_icp_refine + ltr_knn_diff_refined on the orchestrator's own inputs."""
    sess, _ = scenes
    c, q = (s.subset(0, 4) for s in sess[True])
    qp = _perturb(q.poses, 0.3, 1.0)
    G = _orchestrator(c, q, qp, num_knn=2, knn_thr=0.01)
    G.set_icp_refinement(True)
    G.run_step0()
    G.run_step12()
    with F3.ctx() as ctx:
        for s, other, poses in ((0, 1, c.poses), (1, 0, qp)):
            st = G.icp_stats(s)
            scans, off = G.scanset("keyframe_scans_static_projected_", s)
            ss = ctx.scanset_upload(scans, off); ps = ctx.poses_upload(poses, oracle.inverse_poses(poses))
            th = ctx.cloud_upload(G.cloud("map_global_curr_static_", other))
            T, fit, it, ex = ctx.icp_refine(ss, ps, ctx.voxel_centroid(th, 0.4))
            assert _same(T, st["T"]) and np.array_equal(fit, st["fitness"]) and np.array_equal(it, st["iterations"])
            assert np.array_equal(ex, st["exit"]) and np.array_equal(st["accepted"], fit < 1.0)
            co, di = ctx.knn_diff_refined(ss, ps, th, 2, 0.01, T, fit < 1.0)
            for h, member in ((co, "scans_knn_coexist_"), (di, "scans_knn_diff_")):
                a, b = ctx.scanset_download(h), G.scanset(member, s)
                assert _same(a[0], b[0]) and np.array_equal(a[1], b[1]), (s, member)
    G.close()


@pytest.mark.gpu
def test_orchestrator_scanside_removal(scenes):
    sess, _ = scenes
    c, q = (s.subset(0, 4) for s in sess[True])
    G = _orchestrator(c, q, num_knn=3, knn_thr=0.1)
    G.run_step0()
    G.run_step12()
    with F3.ctx() as ctx:
        for crit in (so.MAP, so.SCAN_MINUS_MAP):
            for m_sess, s_sess in ((0, 0), (1, 0), (1, 1)):
                d = (c, q)[s_sess]
                G.scanside_removal(m_sess, s_sess, crit)
                scans, off = G.scanset("keyframe_scans_", s_sess)
                m = G.cloud("map_global_curr_static_", m_sess)
                ss = ctx.scanset_upload(scans, off); ps = ctx.poses_upload(d.poses, oracle.inverse_poses(d.poses)); mh = ctx.cloud_upload(m)
                st, dy = ctx.scanside_split(ss, ps, mh, crit, 3, 0.1)
                for h, member in ((st, "scans_static_"), (dy, "scans_dynamic_")):
                    a, b = ctx.scanset_download(h), G.scanset(member, s_sess)
                    assert _same(a[0], b[0]) and np.array_equal(a[1], b[1]), (crit, m_sess, s_sess, member)
                if (m_sess, s_sess) == (1, 0):
                    exp = so.split_session(scans, off, d.poses, oracle.inverse_poses(d.poses), m, crit, 3, 0.1, L2B, B2L, 1)
                    got = _per_kf(*G.scanset("scans_static_", s_sess))
                    assert all(_same(x, y) for x, y in zip(got, exp[0])), crit
    G.close()


def _step1(c, q, ball=None, adaptive=None):
    G = _orchestrator(c, q, num_knn=2, knn_thr=0.01)
    if ball is not None:
        G.set_map_ball(ball)
    if adaptive is not None:
        G.set_adaptive_threshold(adaptive)
    G.run_step0()
    G.stage("makeGlobalMap")
    M = G.cloud("map_global_curr_", 0)
    G.stage("removeHighDynamicPoints")
    out = (M, G.log(), G.cloud("map_global_curr_static_", 0))
    G.close()
    return out


@pytest.mark.gpu
def test_orchestrator_map_ball_and_adaptive_threshold(scenes):
    """Step 1's removeOnce(2.5) with set_map_ball(R), then with set_adaptive_threshold(0.05): the pass log and the static map equal a
    replay through the Context calls on the orchestrator's own map, and the restatements' flag counts."""
    sess, maps = scenes
    c, q = sess[True]
    inv = oracle.inverse_poses(c.poses)
    radius = _radius(maps["F3"][0], c.poses)
    for kind in ("ball", "adaptive"):
        M, log, static = _step1(c, q, ball=radius if kind == "ball" else None, adaptive=0.05 if kind == "adaptive" else None)
        with F3.ctx() as ctx:
            mh = ctx.cloud_upload(M); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
            if kind == "ball":
                n = ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, radius)
                exp = B.remove_pass(M, c.xyzi, c.offsets, c.poses, inv, oracle.MODE_HD, 2.5, radius, lidar2base=L2B, order=1)
            else:
                n = ctx.remove_pass_adaptive(mh, ss, ps, ltr.MODE_HD, 2.5, 0.05)
                exp = A.remove_pass(M, c.xyzi, c.offsets, inv, oracle.MODE_HD, 2.5, 0.05, lidar2base=L2B, order=1)
            sh, _ = ctx.apply_partition(mh)
            exp_static = ctx.cloud_download(ctx.voxel_centroid(sh, 0.05))
        assert log[0][0] == "removeOnce" and log[0][1] == len(M) and log[0][2] == n == int(exp.sum()), (kind, log[0])
        assert _same(static, exp_static) and _same(static, oracle.voxel(M[exp == 0], 0.05)), kind


@pytest.fixture(scope="module")
def cascade_f3():
    """Sessions 0 -> 1 -> 2 of synth, recorded by the L2B-mounted LiDAR, promoted in memory under F3 with delta maps on."""
    K = 4
    sess = [lidar_session(synth.make_session(s, K, beams=32, az_steps=900)) for s in (0, 1, 2)]
    loaded = [D.pack([removert.voxel_grid(d.scan(k), 0.05)[0] for k in range(d.K)]) for d in sess]
    inv = [oracle.inverse_poses(d.poses) for d in sess]
    G = removert.Removerter(num_knn=2, knn_thr=0.01, lidar2base=L2B, transform_order=1)
    G.set_delta_maps(True)
    G.load_session(0, *loaded[0], sess[0].poses, inv[0])
    gen = []
    for g in (1, 2):
        G.load_session(1, *loaded[g], sess[g].poses, inv[g])
        G.run_step0(); G.run_step12(); G.run_step3()
        gen.append((D.split_sets(*G.scanset("keyframe_scans_pd_", 0)), D.split_sets(*G.scanset("keyframe_scans_strong_nd_", 0))))
        G.cascade_promote_updated()
    yield G, gen, sess[0].poses, D.split_sets(*G.scanset("keyframe_scans_", 0))
    G.close()


@pytest.mark.gpu
def test_orchestrator_delta_maps(cascade_f3):
    G, deltas, poses, live = cascade_f3
    assert G.delta_count() == 2
    G.compose_changes(0, 2)
    pd, nd = D.compose(deltas, 0, 2, 2, 0.01)
    assert all(_same(a, b) for a, b in zip(D.split_sets(*G.scanset("composed_pd_", 0)), pd))
    assert all(_same(a, b) for a, b in zip(D.split_sets(*G.scanset("composed_nd_", 0)), nd))
    assert sum(map(len, pd)) > 0 and sum(map(len, nd)) > 0
    for i in (0, 1, 2):
        G.rollback(i)
        want = D.rollback(live, deltas, i, 2, 0.01)
        got = D.split_sets(*G.scanset("keyframe_scans_restored_", 0))
        assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want)), i
        restored = G.cloud("saved:restored_map")
        assert _same(restored, D.merged_map(want, poses, lidar2base=L2B, order=1)), i


# ================================================================================================================ 5. driver (F3)
def _yaml(tmp_path, out, central=None, query="query", pose_src="central", start=2, end=5, knn=(3, 0.1)):
    central = central or f"{tmp_path}/central/Scans/"
    return ("removert:\n  saveMapPCD: true\n" + f'  save_pcd_directory: "{out}"\n'
            + f'  central_sess_scan_dir: "{central}"\n  central_sess_pose_path: "{tmp_path}/{pose_src}/poses.txt"\n'
            + f'  query_sess_scan_dir: "{tmp_path}/{query}/Scans/"\n  query_sess_pose_path: "{tmp_path}/{query}/poses.txt"\n'
            + "  sequence_vfov: 50\n  sequence_hfov: 360\n"
            + "  ExtrinsicLiDARtoPoseBase: [" + ", ".join(repr(float(v)) for v in L2B.ravel()) + "]\n"
            + f"  keyframe_gap: 1\n  start_idx: {start}\n  end_idx: {end}\n  remove_resolution_list: [2.5]\n  downsample_voxel_size: 0.05\n"
            + f"  num_nn_points_within: {knn[0]}\n  dist_nn_points_within: {knn[1]}\n")


def _write_session(d, s):
    os.makedirs(d / "Scans", exist_ok=True)
    with open(d / "poses.txt", "w") as f:
        for k in range(s.K):
            removert.write_pcd(str(d / "Scans" / f"{k:06d}.pcd"), s.scan(k))
            f.write(" ".join(repr(float(v)) for v in s.poses[k][:3].ravel()) + "\n")


def _drive(tmp_path, tag, args, **kw):
    out = tmp_path / f"out_{tag}"
    cfg = tmp_path / f"params_{tag}.yaml"
    cfg.write_text(_yaml(tmp_path, out, **kw))
    r = subprocess.run([BIN, "--config", str(cfg), "--pcl110"] + args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


def _loaded(tmp_path, sessions):
    """the driver's keyframe selection and pose files, as arrays"""
    c, q = sessions
    kc = removert.parse_keyframes(c.K, 2, 5, 1)
    kq = removert.parse_keyframes_in_roi(q.poses, c.poses[kc], 1)
    out = []
    for s, d, ks in ((0, c, kc), (1, q, kq)):
        xyzi = np.concatenate([d.scan(k) for k in ks]); off = np.concatenate([[0], np.cumsum([len(d.scan(k)) for k in ks])]).astype(np.int64)
        poses = removert.read_poses(str(tmp_path / ("central" if s == 0 else "query") / "poses.txt"))[ks]
        out.append((list(ks), xyzi, off, poses))
    return out


PER_KF = (("scans_updated", "keyframe_scans_updated_"), ("scans_updated_strong", "keyframe_scans_updated_strong_"),
          ("scans_pd", "keyframe_scans_pd_"), ("scans_pd_strong", "keyframe_scans_strong_pd_"), ("scans_nd_strong", "keyframe_scans_strong_nd_"))


ORACLE_SAVED = ["OriginalNoisyCentralMapGlobal", "central_sess_high_dyn", "query_sess_high_dyn", "union_map_queryside", "union_map_centralside",
                "pd_map", "nd_map", "strong_nd_map", "weak_nd_map", "strong_pd_map", "weak_pd_map", "updated_map", "updated_map_strong"]


def _compare_tree(out, saved, per_kf, kc, only=None):
    """every top-level map (or those of `only`) and every per-keyframe scan the driver wrote equals saved(name) / per_kf(member, i), bit for
    bit"""
    names = [f for f in os.listdir(out) if f.endswith(".pcd")]
    assert {"pd_map.pcd", "nd_map.pcd", "updated_map.pcd", "OriginalNoisyCentralMapGlobal.pcd"} <= set(names), names
    if only is not None:
        assert set(only) <= {f[:-4] for f in names}
        names = [n + ".pcd" for n in only]
    for f in names:
        assert _same(removert.read_pcd(str(out / f)), saved(f[:-4])), f
    for sub, member in PER_KF:
        files = sorted(os.listdir(out / sub))
        assert files == [f"{k:06d}.pcd" for k in kc], sub
        for i, fn in enumerate(files):
            assert _same(removert.read_pcd(str(out / sub / fn)), per_kf(member, i)), (sub, fn)


@pytest.fixture(scope="module")
def f3_dataset(tmp_path_factory, scenes):
    tmp = tmp_path_factory.mktemp("f3")
    sess, _ = scenes
    for name, s in zip(("central", "query"), sess[True]):
        _write_session(tmp / name, s)
    return tmp, sess[True]


@pytest.mark.gpu
def test_driver_base_run_matches_the_oracle_and_the_orchestrator(f3_dataset):
    tmp, sessions = f3_dataset
    out = _drive(tmp, "base", [])
    loaded = _loaded(tmp, sessions)
    O = oracle.Removerter(num_knn=3, knn_thr=0.1, lidar2base=L2B, order=1)
    G = removert.Removerter(num_knn=3, knn_thr=0.1, lidar2base=L2B, transform_order=1)
    for s, (ks, xyzi, off, poses) in enumerate(loaded):
        O.load_session(s, xyzi, off, poses, oracle.inverse_poses(poses))
        G.load_session_raw(s, xyzi, off, poses, removert.inverse_poses(poses))
    O.run(step3=True)
    G.run_step0(); G.run_step12(); G.run_step3()
    kc = loaded[0][0]
    _compare_tree(out, lambda n: O.cloud("saved:" + n), lambda m, i: O.cloud(m, 0, i), kc, only=ORACLE_SAVED)
    _compare_tree(out, lambda n: G.cloud("saved:" + n), lambda m, i: _per_kf(*G.scanset(m, 0))[i], kc)
    G.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flag", ["--icp-refinement", "--clean-scans", "--clean-scans=scan-minus-map", "--map-ball=15",
                                  "--adaptive-threshold=0.05"])
def test_driver_features_write_what_the_orchestrator_holds(f3_dataset, flag):
    tmp, sessions = f3_dataset
    tag = flag.strip("-").replace("=", "_")
    out = _drive(tmp, tag, [flag])
    loaded = _loaded(tmp, sessions)
    G = removert.Removerter(num_knn=3, knn_thr=0.1, lidar2base=L2B, transform_order=1)
    if flag == "--icp-refinement":
        G.set_icp_refinement(True)
    elif flag.startswith("--map-ball"):
        G.set_map_ball(15.0)
    elif flag.startswith("--adaptive"):
        G.set_adaptive_threshold(0.05)
    for s, (ks, xyzi, off, poses) in enumerate(loaded):
        G.load_session_raw(s, xyzi, off, poses, removert.inverse_poses(poses))
    G.run_step0(); G.run_step12(); G.run_step3()
    kc = loaded[0][0]
    _compare_tree(out, lambda n: G.cloud("saved:" + n), lambda m, i: _per_kf(*G.scanset(m, 0))[i], kc)
    if flag.startswith("--clean-scans"):
        crit = so.SCAN_MINUS_MAP if flag.endswith("scan-minus-map") else so.MAP
        for s, name in ((0, "central"), (1, "query")):
            G.scanside_removal(s, s, crit)
            ks, _, _, poses = loaded[s]
            for member, sub, kind in (("scans_static_", "scan_static", "Static"), ("scans_dynamic_", "scan_dynamic", "Dynamic")):
                exp = _per_kf(*G.scanset(member, s))
                files = sorted(os.listdir(out / sub / name))
                assert files == [f"{k:06d}.pcd" for k in ks]
                for fn, e in zip(files, exp):
                    assert _same(removert.read_pcd(str(out / sub / name / fn)), e), (sub, name, fn)
                merged = removert.read_pcd(str(out / f"map_{kind.lower()}" / f"{name.capitalize()}{kind}ScansMergedMapGlobal.pcd"))
                assert _same(merged, D.merged_map(exp, poses, lidar2base=L2B, order=1)), (sub, name)
    G.close()


@pytest.mark.gpu
def test_driver_compose_matches_in_memory(tmp_path):
    """Two cascade generations through files under F3, then --compose --pcl110 over both trees == the same deltas composed in memory."""
    import shutil
    K = 4
    for name, s in zip("abc", [lidar_session(synth.make_session(s, K, beams=32, az_steps=900)) for s in (0, 1, 2)]):
        _write_session(tmp_path / name, s)
    kw = dict(pose_src="a", start=0, end=100, knn=(2, 0.01))
    _drive(tmp_path, "g1", [], central=f"{tmp_path}/a/Scans/", query="b", **kw)
    shutil.copytree(tmp_path / "out_g1" / "scans_updated", tmp_path / "central2")
    _drive(tmp_path, "g2", [], central=f"{tmp_path}/central2", query="c", **kw)
    shutil.copytree(tmp_path / "out_g2" / "scans_updated", tmp_path / "central3")
    out = _drive(tmp_path, "g3", [f"--compose={tmp_path}/out_g1,{tmp_path}/out_g2"], central=f"{tmp_path}/central3", query="c", **kw)
    names = sorted(os.listdir(tmp_path / "out_g2" / "scans_pd"))
    idx = [int(n.split(".")[0]) for n in names]
    poses = removert.read_poses(str(tmp_path / "a" / "poses.txt"))[idx]
    live = D.pack([removert.read_pcd(str(tmp_path / "central3" / n)) for n in names])
    G = removert.Removerter(num_knn=2, knn_thr=0.01, lidar2base=L2B, transform_order=1)
    try:
        G.load_session_raw(0, *live, poses, oracle.inverse_poses(poses))
        G.set_delta_maps(True)
        for g in ("out_g1", "out_g2"):
            G.delta_load(*D.pack([removert.read_pcd(str(tmp_path / g / "scans_pd" / n)) for n in names]),
                         *D.pack([removert.read_pcd(str(tmp_path / g / "scans_nd_strong" / n)) for n in names]))
        G.compose_changes(0, 2)
        G.rollback(0)
        for sub, member in (("scans_pd", "composed_pd_"), ("scans_nd_strong", "composed_nd_"), ("scans_restored", "keyframe_scans_restored_")):
            got = D.split_sets(*G.scanset(member, 0))
            for k, n in enumerate(names):
                assert _same(removert.read_pcd(str(out / "composed" / sub / n)), got[k]), (sub, n)
        restored = removert.read_pcd(str(out / "composed" / "restored_map.pcd"))
        assert _same(restored, G.cloud("saved:restored_map"))
        assert _same(restored, D.merged_map(D.split_sets(*G.scanset("keyframe_scans_restored_", 0)), poses, lidar2base=L2B, order=1))
    finally:
        G.close()
