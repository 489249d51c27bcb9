"""The CPU restatement of the ICP refinement (tests/_icp_oracle.py) against independent checks: exit reasons, recovery of a known rigid
error, the rigid solve against a numpy-SVD Umeyama, and the lowest-index tie rule."""
import numpy as np
import pytest

import oracle
import _icp_oracle as io


def _rot(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    R = np.eye(4)
    R[i, i] = c; R[j, j] = c; R[i, j] = -s; R[j, i] = s
    return R


def _umeyama(P, Q):
    pm, qm = P.mean(0), Q.mean(0)
    H = (P - pm).T @ (Q - qm)
    U, _, Vt = np.linalg.svd(H)
    D = np.eye(3)
    D[2, 2] = np.sign(np.linalg.det(Vt.T @ U.T))
    R = Vt.T @ D @ U.T
    return R, qm - R @ pm, H, pm, qm


@pytest.mark.parametrize("seed", range(6))
def test_rigid_solve_matches_svd_umeyama(seed):
    rng = np.random.default_rng(seed)
    P = rng.normal(size=(40 + 10 * seed, 3)) * [3, 2, 1]
    E = _rot(0, rng.uniform(-40, 40)) @ _rot(1, rng.uniform(-40, 40)) @ _rot(2, rng.uniform(-180, 180))
    Q = P @ E[:3, :3].T + rng.normal(size=3) * 5 + rng.normal(scale=0.05, size=P.shape)
    Ru, tu, H, pm, qm = _umeyama(P, Q)
    R, t = io.horn_rigid(H.reshape(9), list(pm), list(qm))
    assert np.abs(np.array(R).reshape(3, 3) - Ru).max() < 1e-6
    assert np.abs(np.array(t) - tu).max() < 1e-6


def test_rigid_solve_reflection_case():
    """A mirrored target: the unconstrained optimum is a reflection; SVD with the det fix and Horn's quaternion both give the best proper
    rotation."""
    rng = np.random.default_rng(11)
    P = rng.normal(size=(60, 3)) * [4, 2, 1]
    Q = P * [1, 1, -1] + rng.normal(scale=0.02, size=P.shape)
    Ru, tu, H, pm, qm = _umeyama(P, Q)
    U, _, Vt = np.linalg.svd(H)
    assert np.linalg.det(Vt.T @ U.T) < 0, "the input must need the reflection fix"
    R, t = io.horn_rigid(H.reshape(9), list(pm), list(qm))
    R = np.array(R).reshape(3, 3)
    assert abs(np.linalg.det(R) - 1.0) < 1e-12
    assert np.abs(R - Ru).max() < 1e-6
    assert np.abs(np.array(t) - tu).max() < 1e-6


def test_nearest_neighbour_ties_take_the_lowest_index():
    ax = np.arange(-3, 4, dtype=np.float32) * 0.5
    g = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    t = np.concatenate([g, np.zeros((len(g), 1))], 1).astype(np.float32)
    t = np.concatenate([t[::-1], t])            # every lattice point twice, the copies far apart in index
    tgt = io.Target(t)
    q = (g + np.float32(0.25)).astype(np.float32)   # midway between lattice points: up to 8 points at the same distance, each twice
    d, idx = tgt.nn(q)
    for i in range(len(q)):
        dd = io.l2_simple(q[i], t)
        assert d[i] == dd.min()
        assert idx[i] == np.nonzero(dd == dd.min())[0].min()


def _scene(K=2):
    import synth
    c, _ = synth.make_pair(K, beams=32, az_steps=900)
    m = oracle.voxel(np.concatenate([oracle.transform(c.scan(k), c.poses[k]) for k in range(c.K)]), 0.4)
    return c, m


@pytest.mark.parametrize("trans,deg", [(0.05, 0.2), (0.3, 1.0), (1.0, 3.0)])
def test_known_rigid_error_is_recovered(trans, deg):
    """Keyframe poses carrying a known rigid error E in the sensor frame (pose @ E) are registered to the session's own 0.4 m map; the
    residual is final @ pose @ E @ pose^-1.  A 0.05 m / 0.2 degree error is removed to within 0.02 m and 0.05 degrees.  Larger ones are
    reduced, not always removed: point-to-point ICP on 0.4 m centroids stops on the 1e-6 increment test, and the synthetic street repeats
    every few metres (0.3 m / 1 degree leaves at most 0.31 m and 0.31 degrees, 1 m / 3 degrees at most 0.97 m and 1.3 degrees here).
    Every refined keyframe is accepted (fitness < 1.0)."""
    c, m = _scene()
    E = _rot(2, deg) @ _rot(0, deg / 3)
    E[:3, 3] = np.array([1.0, -0.6, 0.2]) * trans
    poses = np.stack([p @ E for p in c.poses])
    T, fit, it, ex = io.refine_session(c.xyzi, c.offsets, poses, m)
    ang0 = np.rad2deg(np.arccos((np.trace(E[:3, :3]) - 1) / 2))
    for k in range(c.K):
        err = T[k].astype(np.float64) @ poses[k] @ np.linalg.inv(c.poses[k])
        ang = np.rad2deg(np.arccos(np.clip((np.trace(err[:3, :3]) - 1) / 2, -1, 1)))
        assert ang < 0.5 * ang0, (k, err, it[k], ex[k])
        if trans <= 0.05:
            assert np.abs(err[:3, 3]).max() < 0.02 and ang < 0.05, (k, err, it[k], ex[k])
    assert (fit < 1.0).all() and (it > 1).all()


def test_every_exit_reason_is_reached():
    c, m = _scene(1)
    scan = c.scan(0)
    off = np.array([0, len(scan)], np.int64)
    E = _rot(2, 1.0)
    E[:3, 3] = [0.2, 0.1, 0.0]
    poses = (E @ c.poses[0])[None]
    # 1: the iteration cap
    assert io.refine_session(scan, off, poses, m, max_iterations=2)[3][0] == io.ITERATIONS
    # 2: the default run converges on a small increment
    assert io.refine_session(scan, off, poses, m)[3][0] == io.TRANSFORM
    # 3 / 4: with the increment test switched off the MSE change decides, absolute first
    assert io.refine_session(scan, off, poses, m, transformation_epsilon=0.0, mse_threshold_absolute=1e-3)[3][0] == io.ABS_MSE
    assert io.refine_session(scan, off, poses, m, transformation_epsilon=0.0, euclidean_fitness_epsilon=1e-2)[3][0] == io.REL_MSE
    # 5: fewer than three correspondences (empty, one and two source points) -- identity, DBL_MAX fitness without points
    two = np.array([[1, 2, 3, 0], [5, 5, 1, 0]], np.float32)
    T, fit, it, ex = io.refine_session(np.concatenate([two[:0], two[:1], two]), np.array([0, 0, 1, 3]), np.stack([np.eye(4)] * 3), m)
    assert list(ex) == [io.NO_CORRESPONDENCES] * 3 and list(it) == [0, 0, 0]
    assert fit[0] == io.DBL_MAX and np.isfinite(fit[1]) and (T == np.eye(4, dtype=np.float32)).all()
    # 5 again: every pair beyond the correspondence distance
    assert io.refine_session(scan, off, poses, m, max_correspondence_distance=1e-4)[3][0] == io.NO_CORRESPONDENCES


def test_reduction_shape():
    """tree_sums: B sequential partials then the binary tree -- exact on integers, and not the naive left-to-right sum in general."""
    x = np.arange(1000, dtype=np.float64)
    assert io.tree_sums(x[:, None])[0] == x.sum()
    rng = np.random.default_rng(5)
    y = rng.normal(size=5000) * 10.0 ** rng.integers(-8, 8, 5000)
    s = 0.0
    part = [0.0] * io.B
    for i, v in enumerate(y):
        part[i % io.B] += v
    stride = io.B // 2
    while stride:
        for j in range(stride):
            part[j] += part[j + stride]
        stride //= 2
    s = part[0]
    assert io.tree_sums(y[:, None])[0] == s
