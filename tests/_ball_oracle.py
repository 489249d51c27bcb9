"""CPU restatement of the remove / revert / ND / PD pass on ball subsets of the map (test infrastructure, not product code).

takeGlobalMapSubsetWithinBall (ltremovert/src/Removerter.cpp:415-427, behind kUseSubsetMapCloud / kBallSize, Removerter.h:46-48) as the
contract of ltr_remove_pass_ball fixes it: keyframe k sees the map points i with d2 < r2, where d2 = ((dx dx) + dy dy) + dz dz in float32
with dx = fl(x_i - c_k.x), c_k the float32-rounded translation column of poses[k], and r2 = (float)(R * R) in double (FLANN's L2_Simple
distance and strict radius test, as PCL's KdTreeFLANN::radiusSearch drives it).  The subset keeps map order.  The flags are the OR over
the keyframes of the single-keyframe pass on the subset, mapped back to map indices.  The single-keyframe pass is the oracle's own
(oracle.remove_pass, or tests/_adaptive_oracle.py for the adaptive threshold), so the membership rule is the only new part; numpy's
elementwise float32 operations round exactly as the contract does.
"""
import numpy as np

import oracle
import _adaptive_oracle

F32 = np.float32


def centres(poses):
    """(K, 3) float32: the translation column of each pose, rounded to float32 (the ball centres)."""
    return np.asarray(poses, np.float64)[:, :3, 3].astype(F32)


def radius2(radius):
    """r2 = (float)((double)R * (double)R) (inf beyond FLT_MAX)."""
    with np.errstate(over="ignore"):
        return F32(np.float64(F32(radius)) * np.float64(F32(radius)))


def sq_dist(xyz, c):
    """d2 of every point from centre c, in float32 without contraction (NaN / inf stay non-finite)."""
    p = np.asarray(xyz, F32)[:, :3]
    c = np.asarray(c, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        dx, dy, dz = p[:, 0] - c[0], p[:, 1] - c[1], p[:, 2] - c[2]
        return (dx * dx + dy * dy) + dz * dz


def members(xyz, c, radius):
    """bool (N,): the points of the ball of `radius` around c (d2 < r2; NaN compares false)."""
    with np.errstate(invalid="ignore"):
        return sq_dist(xyz, c) < radius2(radius)


def remove_pass(map_xyzi, scans_xyzi, offsets, poses, inv_poses, mode, alpha, radius, thres=0.1, coeff=0.0, lidar2base=oracle.IDENTITY,
                order=0):
    """flags (N,) uint8: the OR over the keyframes of the single-keyframe pass on the keyframe's ball subset.  The ball is centred on the
    pose (the base), whatever the extrinsic; lidar2base and the transform order only reach the single-keyframe pass's projection."""
    m = np.ascontiguousarray(map_xyzi, F32)
    s = np.ascontiguousarray(scans_xyzi, F32)
    flags = np.zeros(len(m), np.uint8)
    cs = centres(poses)
    for k in range(len(offsets) - 1):
        idx = np.flatnonzero(members(m, cs[k], radius))
        if len(idx) == 0:
            continue
        scan = s[offsets[k]:offsets[k + 1]]
        off = np.array([0, len(scan)], np.int64)
        if coeff:
            f = _adaptive_oracle.remove_pass(m[idx], scan, off, inv_poses[k:k + 1], mode, alpha, coeff, lidar2base=lidar2base, order=order)
        else:
            f = oracle.remove_pass(m[idx], scan, off, inv_poses[k:k + 1], mode, alpha, thres, lidar2base=lidar2base, order=order)
        flags[idx[f != 0]] = 1
    return flags
