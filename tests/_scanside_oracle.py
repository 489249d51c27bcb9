"""CPU restatement of scan-side removal (test infrastructure, not product code).

Removerter::removeDynamicPointsOfScanByKnn, both overloads (ltremovert/src/Removerter.cpp:1019-1069 "map", 1071-1123 "scan minus map"),
as scansideRemovalForEachScan (Removerter.cpp:1253-1310) calls it per keyframe.  Built from the oracle's primitives only: its
pcl::transformPointCloud restatement (oracle.transform) and its exact k-NN (oracle.knn_dists: the k smallest FLANN L2_Simple squared
distances, ascending, +inf past the target's size), which already returns exact values, not threshold decisions.
"""
import numpy as np

import oracle

MAP, SCAN_MINUS_MAP = 0, 1


def _is_identity(m):
    return np.array_equal(np.asarray(m, np.float64), np.eye(4))


def knn_avg(q_xyzi, t_xyzi, k):
    """(float)(accumulate(k smallest squared distances, 0.0)) / float(k) per query (Removerter.cpp:1051-1053, 1096-1098): the double sum
    runs in ascending order over min(k, len(target)) values and is still divided by k."""
    d = oracle.knn_dists(q_xyzi, t_xyzi, k)
    s = np.zeros(len(d), np.float64)
    for j in range(min(k, len(t_xyzi))):
        s = s + d[:, j].astype(np.float64)
    return (s.astype(np.float32) / np.float32(k)).astype(np.float32)


def local2global(scan_xyzi, pose, lidar2base=oracle.IDENTITY, order=0):
    """utility.cpp:160-168 (3-argument overload): lidar2base, then the pose, f32 rounding after each step.  An exactly-identity
    extrinsic step is skipped, as the device does (it is exact)."""
    g = np.asarray(scan_xyzi, np.float32)
    if not _is_identity(lidar2base):
        g = oracle.transform(g, lidar2base, order)
    return oracle.transform(g, pose, order)


def global2local(xyzi, inv_pose, base2lidar=oracle.IDENTITY, order=0):
    """utility.cpp:194-202: inverse pose, then base2lidar."""
    out = oracle.transform(np.asarray(xyzi, np.float32), inv_pose, order)
    if not _is_identity(base2lidar):
        out = oracle.transform(out, base2lidar, order)
    return out


def split_scan(scan_xyzi, pose, inv_pose, map_xyzi, criterion, k, thr, lidar2base=oracle.IDENTITY, base2lidar=oracle.IDENTITY, order=0):
    """(static_local, dynamic_local, static_mask) of one keyframe, both parts in input order."""
    if len(map_xyzi) == 0:
        raise ValueError("empty map (PCL's nearestKSearch asserts on an empty tree)")
    g = local2global(scan_xyzi, pose, lidar2base, order)
    thr = np.float32(thr)
    if len(g) == 0:
        mask = np.zeros(0, bool)
    else:
        avg_map = knn_avg(g, map_xyzi, k)
        if criterion == MAP:
            mask = np.abs(avg_map) < thr                                  # Removerter.cpp:1056
        else:
            avg_scan = knn_avg(g, g, k)
            mask = np.abs((avg_scan - avg_map).astype(np.float32)) < thr  # Removerter.cpp:1107, f32 subtraction
    return global2local(g[mask], inv_pose, base2lidar, order), global2local(g[~mask], inv_pose, base2lidar, order), mask


def split_session(xyzi, offsets, poses, inv_poses, map_xyzi, criterion, k, thr, lidar2base=oracle.IDENTITY, base2lidar=oracle.IDENTITY,
                  order=0, pose_offset=0):
    """Per-keyframe (static list, dynamic list) of scansideRemovalForEachScan for one (map, scan) session pair."""
    st, dy = [], []
    for kf in range(len(offsets) - 1):
        s, d, _ = split_scan(xyzi[offsets[kf]:offsets[kf + 1]], poses[pose_offset + kf], inv_poses[pose_offset + kf], map_xyzi, criterion, k,
                             thr, lidar2base, base2lidar, order)
        st.append(s)
        dy.append(d)
    return st, dy
