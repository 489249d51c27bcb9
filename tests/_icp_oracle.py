"""CPU restatement of the ICP refinement of the low-dynamic kNN diff (test infrastructure, not product code).

Session::partitionLowDynamicPointsOfScanByKnn with `useICPrefinement` on (ltremovert/src/Session.cpp:549-584) under the contract of
DESIGN.md §5.2 / lt_mapper_b200/csrc/icp.cu: PCL's IterativeClosestPoint control flow, this project's arithmetic.  Built on the oracle's
pcl::transformPointCloud (oracle.transform), octreeDownsampling (oracle.voxel) and exact k-NN (oracle.knn_dists, the nearest f32 L2_Simple
value); the lowest target index at that value comes from a candidate set of a scipy k-d tree, checked in f32.  The rigid solve is plain
Python floats (IEEE double, no FMA); every sum has the device's reduction shape (B sequential partials, then a binary tree).
"""
import sys

import numpy as np
from scipy.spatial import cKDTree

import oracle
import _scanside_oracle as so

B = 256               # kIcpThreads
JACOBI_SWEEPS = 10    # kJacobiSweeps
ITERATIONS, TRANSFORM, ABS_MSE, REL_MSE, NO_CORRESPONDENCES = 1, 2, 3, 4, 5
DBL_MAX = sys.float_info.max
DEFAULTS = dict(max_correspondence_distance=150.0, max_iterations=100, transformation_epsilon=1e-6, euclidean_fitness_epsilon=1e-6,
                mse_threshold_absolute=1e-12, min_correspondences=3, source_leaf=0.4)


def l2_simple(q, p):
    """FLANN L2_Simple in f32: ((dx*dx) + dy*dy) + dz*dz, dx = query - point."""
    d = (np.asarray(q, np.float32)[..., :3] - np.asarray(p, np.float32)[..., :3]).astype(np.float32)
    return ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(np.float32)


def tree_sums(cols):
    """Column sums of cols (n, m) float64 in the device's shape: partial[j] = sequential sum of rows j, j + B, ...; then the tree."""
    cols = np.asarray(cols, np.float64)
    n, m = cols.shape
    rounds = -(-n // B)
    pad = np.zeros((max(rounds, 1) * B, m))
    pad[:n] = cols
    part = np.zeros((B, m))
    for r in range(rounds):
        part = part + pad[r * B:(r + 1) * B]
    s = B // 2
    while s:
        part[:s] = part[:s] + part[s:2 * s]
        s //= 2
    return [float(v) for v in part[0]]


def apply(T, xyz):
    """f32 rigid transform ((m0 x + m1 y) + m2 z) + m3 of (n, >=3) points; returns (n, 3) float32."""
    T = np.asarray(T, np.float32)
    p = np.asarray(xyz, np.float32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((T[r, 0] * x + T[r, 1] * y) + T[r, 2] * z) + T[r, 3] for r in range(3)], 1).astype(np.float32)


def compose(T, F):
    """T F as an f32 4x4 product, ((T[r][0] F[0][c] + T[r][1] F[1][c]) + T[r][2] F[2][c]) + T[r][3] F[3][c]."""
    out = np.empty((4, 4), np.float32)
    for r in range(4):
        for c in range(4):
            out[r, c] = ((T[r, 0] * F[0, c] + T[r, 1] * F[1, c]) + T[r, 2] * F[2, c]) + T[r, 3] * F[3, c]
    return out


def horn_rigid(H, pm, qm):
    """(R row-major 3x3, t) maximising sum q.(R p) over proper rotations: Horn's quaternion from cyclic Jacobi on his 4x4 matrix N(H).
    H[3a + b] = sum (p_a - pm_a)(q_b - qm_b)."""
    Sxx, Sxy, Sxz, Syx, Syy, Syz, Szx, Szy, Szz = [float(v) for v in H]
    A = [[0.0] * 4 for _ in range(4)]
    A[0][0] = (Sxx + Syy) + Szz
    A[1][1] = (Sxx - Syy) - Szz
    A[2][2] = (-Sxx + Syy) - Szz
    A[3][3] = (-Sxx - Syy) + Szz
    A[0][1] = A[1][0] = Syz - Szy
    A[0][2] = A[2][0] = Szx - Sxz
    A[0][3] = A[3][0] = Sxy - Syx
    A[1][2] = A[2][1] = Sxy + Syx
    A[1][3] = A[3][1] = Szx + Sxz
    A[2][3] = A[3][2] = Syz + Szy
    V = [[1.0 if r == c else 0.0 for c in range(4)] for r in range(4)]
    for _ in range(JACOBI_SWEEPS):
        for p, q in ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)):
            apq = A[p][q]
            if apq == 0.0:
                continue
            theta = (A[q][q] - A[p][p]) / (2.0 * apq)
            t = 1.0 / (abs(theta) + _sqrt(theta * theta + 1.0))
            if theta < 0.0:
                t = -t
            c = 1.0 / _sqrt(t * t + 1.0)
            s = t * c
            for r in range(4):
                if r in (p, q):
                    continue
                arp, arq = A[r][p], A[r][q]
                A[r][p] = A[p][r] = c * arp - s * arq
                A[r][q] = A[q][r] = s * arp + c * arq
            app, aqq = A[p][p], A[q][q]
            A[p][p] = app - t * apq
            A[q][q] = aqq + t * apq
            A[p][q] = A[q][p] = 0.0
            for r in range(4):
                vrp, vrq = V[r][p], V[r][q]
                V[r][p] = c * vrp - s * vrq
                V[r][q] = s * vrp + c * vrq
    m = 0
    for j in range(1, 4):
        if A[j][j] > A[m][m]:
            m = j
    w, x, y, z = V[0][m], V[1][m], V[2][m], V[3][m]
    nrm = _sqrt(((w * w + x * x) + y * y) + z * z)
    w, x, y, z = w / nrm, x / nrm, y / nrm, z / nrm
    ww, xx, yy, zz = w * w, x * x, y * y, z * z
    wx, wy, wz, xy, xz, yz = w * x, w * y, w * z, x * y, x * z, y * z
    R = [((ww + xx) - yy) - zz, 2.0 * (xy - wz), 2.0 * (xz + wy),
         2.0 * (xy + wz), ((ww - xx) + yy) - zz, 2.0 * (yz - wx),
         2.0 * (xz - wy), 2.0 * (yz + wx), ((ww - xx) - yy) + zz]
    t = [qm[a] - ((R[3 * a] * pm[0] + R[3 * a + 1] * pm[1]) + R[3 * a + 2] * pm[2]) for a in range(3)]
    return R, t


def _sqrt(v):
    return float(np.sqrt(np.float64(v)))   # IEEE correctly rounded, as __dsqrt_rn


class Target:
    """The fixed ICP target: nearest f32 L2_Simple value (oracle.knn_dists) and the lowest index at that value."""

    def __init__(self, xyzi):
        self.t = np.ascontiguousarray(np.asarray(xyzi, np.float32).reshape(-1, 4))
        self.tree = cKDTree(self.t[:, :3].astype(np.float64))

    def nn(self, q):
        q = np.ascontiguousarray(np.asarray(q, np.float32)[:, :3])
        n = len(q)
        if n == 0:
            return np.zeros(0, np.float32), np.zeros(0, np.int64)
        qx = np.concatenate([q, np.zeros((n, 1), np.float32)], 1)
        d = oracle.knn_dists(qx, self.t, 1)[:, 0]
        r = np.sqrt(d.astype(np.float64)) * (1 + 1e-3) + 1e-6   # every point at f32 distance d lies inside
        k = min(8, len(self.t))
        dist, idx = self.tree.query(q.astype(np.float64), k=k)
        dist, idx = dist.reshape(n, k), idx.reshape(n, k)
        dd = l2_simple(q[:, None, :], self.t[idx])
        hit = (dd == d[:, None]) & (dist <= r[:, None])
        out = np.where(hit, idx, np.iinfo(np.int64).max).min(1)
        assert hit.any(1).all(), "no candidate at the nearest value"
        for i in np.nonzero((dist <= r[:, None]).all(1) & (k < len(self.t)))[0]:
            # possibly more points at the nearest value than the k nearest: take every point of the ball
            cand = np.asarray(self.tree.query_ball_point(q[i].astype(np.float64), r[i]), np.int64)
            out[i] = cand[l2_simple(q[i], self.t[cand]) == d[i]].min()
        return d, out


def icp(src_xyzi, tgt, **params):
    """One keyframe: (final T (4,4) float32, fitness, iterations, exit reason).  src = the keyframe's 0.4 m global source, tgt a Target."""
    p = dict(DEFAULTS, **params)
    P0 = np.asarray(src_xyzi, np.float32).reshape(-1, 4)[:, :3].copy()
    n = len(P0)
    w = P0.copy()
    F = np.eye(4, dtype=np.float32)
    prev = DBL_MAX
    it = ex = 0
    max_d2 = float(p["max_correspondence_distance"]) * float(p["max_correspondence_distance"])
    rot_thr = 1.0 - float(p["transformation_epsilon"])
    while True:
        d, j = tgt.nn(w)
        valid = d.astype(np.float64) <= max_d2
        cnt = int(valid.sum())
        if cnt < p["min_correspondences"]:
            ex = NO_CORRESPONDENCES
            break
        Q = tgt.t[j, :3] if n else np.zeros((0, 3), np.float32)
        cols = np.stack([w[:, 0], w[:, 1], w[:, 2], Q[:, 0], Q[:, 1], Q[:, 2], d], 1).astype(np.float64)
        sums = tree_sums(np.where(valid[:, None], cols, 0.0))
        pm = [sums[a] / cnt for a in range(3)]
        qm = [sums[3 + a] / cnt for a in range(3)]
        mse = sums[6] / cnt
        dp = w.astype(np.float64) - np.array(pm)
        dq = Q.astype(np.float64) - np.array(qm)
        hc = np.stack([dp[:, r] * dq[:, c] for r in range(3) for c in range(3)], 1)
        H = tree_sums(np.where(valid[:, None], hc, 0.0))
        R, t = horn_rigid(H, pm, qm)
        T = np.eye(4, dtype=np.float32)
        for r in range(3):
            for c in range(3):
                T[r, c] = np.float32(R[3 * r + c])
            T[r, 3] = np.float32(t[r])
        F = compose(T, F)
        it += 1
        cos_angle = 0.5 * float((T[0, 0] + T[1, 1] + T[2, 2]) - np.float32(1.0))
        tsq = float((T[0, 3] * T[0, 3] + T[1, 3] * T[1, 3]) + T[2, 3] * T[2, 3])
        dmse = abs(mse - prev)
        if it >= p["max_iterations"]:
            ex = ITERATIONS
        elif cos_angle >= rot_thr and tsq <= p["transformation_epsilon"]:
            ex = TRANSFORM
        elif dmse < p["mse_threshold_absolute"]:
            ex = ABS_MSE
        elif dmse / prev < p["euclidean_fitness_epsilon"]:
            ex = REL_MSE
        prev = mse
        w = apply(T, w)
        if ex:
            break
    return F, fitness(P0, F, tgt), it, ex


def fitness(src_xyz, F, tgt):
    """getFitnessScore(DBL_MAX): mean nearest d2 of the source moved by F, DBL_MAX without points."""
    if len(src_xyz) == 0:
        return DBL_MAX
    d, _ = tgt.nn(apply(F, src_xyz))
    ok = d.astype(np.float64) <= DBL_MAX
    s = tree_sums(np.where(ok, d.astype(np.float64), 0.0)[:, None])[0]
    c = int(ok.sum())
    return s / c if c else DBL_MAX


def global_scan(scan_xyzi, pose, base2lidar=oracle.IDENTITY, order=0):
    """scan_global as ltr_knn_diff moves a scan: base2lidar (as written at Session.cpp:545), then the pose."""
    return so.local2global(scan_xyzi, pose, base2lidar, order)


def refine_session(xyzi, offsets, poses, target_down, base2lidar=oracle.IDENTITY, order=0, pose_offset=0, **params):
    """ltr_icp_refine: per-keyframe (T (K,4,4) float32, fitness (K,), iterations (K,), exit (K,))."""
    p = dict(DEFAULTS, **params)
    if len(target_down) == 0:
        raise ValueError("empty ICP target")
    tgt = Target(target_down)
    K = len(offsets) - 1
    T = np.zeros((K, 4, 4), np.float32)
    fit = np.zeros(K)
    its = np.zeros(K, np.int32)
    exs = np.zeros(K, np.int32)
    for kf in range(K):
        g = global_scan(xyzi[offsets[kf]:offsets[kf + 1]], poses[pose_offset + kf], base2lidar, order)
        src = oracle.voxel(g, p["source_leaf"]) if len(g) else np.zeros((0, 4), np.float32)
        T[kf], fit[kf], its[kf], exs[kf] = icp(src, tgt, **params)
    return T, fit, its, exs


def knn_diff_refined(xyzi, offsets, poses, inv_poses, target, k, thr, T, accepted, base2lidar=oracle.IDENTITY, order=0, pose_offset=0):
    """ltr_knn_diff_refined: per-keyframe (coexist list, diff list) in the LiDAR frame; accepted keyframes are moved by T[kf] first."""
    co, di = [], []
    thr = np.float32(thr)
    for kf in range(len(offsets) - 1):
        g = global_scan(xyzi[offsets[kf]:offsets[kf + 1]], poses[pose_offset + kf], base2lidar, order)
        if accepted[kf] and len(g):
            g = np.concatenate([apply(T[kf], g), g[:, 3:4]], 1).astype(np.float32)
        mask = np.abs(so.knn_avg(g, target, k)) < thr if len(g) else np.zeros(0, bool)
        co.append(so.global2local(g[mask], inv_poses[pose_offset + kf], base2lidar, order))
        di.append(so.global2local(g[~mask], inv_poses[pose_offset + kf], base2lidar, order))
    return co, di
