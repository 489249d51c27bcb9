"""The CPU restatement of scan-side removal with ICP fine registration (tests/_scanside_reg_oracle.py): it reduces to the plain scan-side
split when nothing is accepted, its ICP source is the kNN diff's with the identity extrinsic, and a registration that undoes a known pose
error turns the points the error pushed off the map back into static points."""
import numpy as np
import pytest

import oracle
import _icp_oracle as io
import _scanside_oracle as so
import _scanside_reg_oracle as sro

L2B = np.array([[np.cos(0.05), 0, np.sin(0.05), 0.3], [0, 1, 0, -0.02], [-np.sin(0.05), 0, np.cos(0.05), 1.1], [0, 0, 0, 1]])


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("criterion", [so.MAP, so.SCAN_MINUS_MAP])
@pytest.mark.parametrize("extrinsic", [False, True])
def test_every_keyframe_rejected_is_the_plain_split(small_pair, small_maps, criterion, extrinsic):
    c = small_pair[0].subset(0, 2)
    l2b = L2B if extrinsic else oracle.IDENTITY
    b2l = oracle.inverse4x4(L2B) if extrinsic else oracle.IDENTITY
    inv = oracle.inverse_poses(c.poses)
    T = np.tile(np.eye(4, dtype=np.float32), (c.K, 1, 1))
    T[:, 0, 3] = 0.5                                    # a transform that would move the points, were any keyframe accepted
    got = sro.split_session_refined(c.xyzi, c.offsets, c.poses, inv, small_maps[1], criterion, 3, 0.1, T, np.zeros(c.K, bool), l2b, b2l)
    exp = so.split_session(c.xyzi, c.offsets, c.poses, inv, small_maps[1], criterion, 3, 0.1, l2b, b2l)
    for part in range(2):
        assert len(got[part]) == c.K
        for kf in range(c.K):
            assert _same(got[part][kf], exp[part][kf]), (part, kf)
    moved = sro.split_session_refined(c.xyzi, c.offsets, c.poses, inv, small_maps[1], criterion, 3, 0.1, T, np.ones(c.K, bool), l2b, b2l)
    assert not all(_same(moved[0][kf], exp[0][kf]) for kf in range(c.K))


def test_icp_source_with_the_identity_extrinsic_is_the_knn_diffs(small_pair):
    c = small_pair[1]
    for kf in range(3):
        scan, pose = c.scan(kf), c.poses[kf]
        assert _same(sro.source(scan, pose), oracle.voxel(io.global_scan(scan, pose), 0.4)), kf
    # with an extrinsic the two paths move the scan by different matrices (lidar2base here, base2lidar there)
    scan, pose = c.scan(0), c.poses[0]
    assert not _same(sro.source(scan, pose, L2B), oracle.voxel(io.global_scan(scan, pose, oracle.inverse4x4(L2B)), 0.4))


def _rot_z(deg):
    a = np.deg2rad(deg)
    R = np.eye(4)
    R[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    return R


def test_registration_undoes_a_known_pose_error():
    """200 Gaussian blobs of points (0.3 m spread); the scan is every second map point seen from the identity pose, but its recorded pose
    carries 0.3 m / 1 degree of error.  Unregistered, the error moves most points more than 0.1 m away from every map point, so under
    the "map" criterion (k = 1, 0.01 m^2) most points are dynamic; registered, the keyframe is accepted and nearly every point is static."""
    rng = np.random.default_rng(7)
    centres = np.c_[rng.uniform(-10, 10, (200, 2)), rng.uniform(0, 4, 200)]
    pts = (centres[:, None, :] + rng.normal(0, 0.3, (200, 150, 3))).reshape(-1, 3)
    m = np.c_[pts, np.zeros(len(pts))].astype(np.float32)
    scan = m[::2].copy()
    offsets = np.array([0, len(scan)], np.int64)
    err = _rot_z(1.0)
    err[:3, 3] = [0.3, 0.2, 0.15]
    poses = err[None]
    inv = oracle.inverse_poses(poses)
    (st, dy), (T, fit, its, exs, acc) = sro.removal_registered(scan, offsets, poses, inv, m, so.MAP, 1, 0.01)
    assert acc[0] and fit[0] < 1.0 and its[0] > 1
    plain_st, _ = so.split_session(scan, offsets, poses, inv, m, so.MAP, 1, 0.01)
    n = len(scan)
    assert len(st[0]) + len(dy[0]) == n
    assert len(plain_st[0]) < 0.5 * n, len(plain_st[0])
    assert len(st[0]) > 0.95 * n, len(st[0])
    # the registration is close to the inverse of the error
    assert np.abs(T[0].astype(np.float64) @ err - np.eye(4)).max() < 0.02
    # rejecting it gives the plain split back
    rej = sro.split_session_refined(scan, offsets, poses, inv, m, so.MAP, 1, 0.01, T, [False])
    assert _same(rej[0][0], plain_st[0])
