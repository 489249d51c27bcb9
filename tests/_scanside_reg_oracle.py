"""CPU restatement of scan-side removal between sessions with ICP fine registration (test infrastructure, not product code).

scansideRemovalForEachScan with isFineRegistration (ltremovert/src/Removerter.cpp:1295-1297) and its per-keyframe body
removeDynamicPointsOfScanByKnnBtnSession (:950-1017), under the accept rule of Session.cpp:571-579 (DESIGN.md §5.4).  Composed from the
existing restatements, each rule stated once there: the registration is _icp_oracle.refine_session with lidar2base as its step-1
extrinsic (its global_scan is _scanside_oracle.local2global, the scan-side transform); accept iff fitness < 1.0 (:978); the split is
_scanside_oracle.split_scan, on the scan itself for a rejected keyframe and on the registered global points for an accepted one.
"""
import numpy as np

import oracle
import _icp_oracle as io
import _scanside_oracle as so


def source(scan_xyzi, pose, lidar2base=oracle.IDENTITY, order=0, leaf=io.DEFAULTS["source_leaf"]):
    """A keyframe's ICP source: its global scan as scan-side removal moves it, octree-downsampled at `leaf` (Removerter.cpp:962-964)."""
    g = io.global_scan(scan_xyzi, pose, lidar2base, order)
    return oracle.voxel(g, leaf) if len(g) else np.zeros((0, 4), np.float32)


def register_session(xyzi, offsets, poses, target_down, lidar2base=oracle.IDENTITY, order=0, pose_offset=0, **params):
    """ltr_icp_refine_scanside: per-keyframe (T (K,4,4) float32, fitness (K,), iterations (K,), exit (K,))."""
    return io.refine_session(xyzi, offsets, poses, target_down, lidar2base, order, pose_offset, **params)


def split_session_refined(xyzi, offsets, poses, inv_poses, map_xyzi, criterion, k, thr, T, accepted, lidar2base=oracle.IDENTITY,
                          base2lidar=oracle.IDENTITY, order=0, pose_offset=0):
    """ltr_scanside_split_refined: per-keyframe (static list, dynamic list) in the LiDAR frame.  A rejected keyframe is split as
    _scanside_oracle.split_session splits it.  An accepted one's global points are moved by T[kf] in f32 (_icp_oracle.apply) and handed to
    split_scan as the "scan" of an identity pose with an identity extrinsic: that forward step returns every finite coordinate unchanged
    (x * 1 + 0 is exact in double) except that it may turn a -0.0 into +0.0, which neither the squared distances nor global2local (whose
    sums meet the pose's non-zero terms) can tell apart; search and relocalisation then use the keyframe's own inv_pose and base2lidar."""
    st, dy = [], []
    for kf in range(len(offsets) - 1):
        scan = xyzi[offsets[kf]:offsets[kf + 1]]
        pose, inv = poses[pose_offset + kf], inv_poses[pose_offset + kf]
        if accepted[kf] and len(scan):
            g = so.local2global(scan, pose, lidar2base, order)
            g = np.concatenate([io.apply(T[kf], g), g[:, 3:4]], 1).astype(np.float32)
            s, d, _ = so.split_scan(g, oracle.IDENTITY, inv, map_xyzi, criterion, k, thr, oracle.IDENTITY, base2lidar, order)
        else:
            s, d, _ = so.split_scan(scan, pose, inv, map_xyzi, criterion, k, thr, lidar2base, base2lidar, order)
        st.append(s)
        dy.append(d)
    return st, dy


def removal_registered(xyzi, offsets, poses, inv_poses, map_static, criterion, k, thr, lidar2base=oracle.IDENTITY,
                       base2lidar=oracle.IDENTITY, order=0, pose_offset=0):
    """ltrh_scanside_removal_registered for one (map, scan) session pair: ((static list, dynamic list), (T, fitness, iterations, exit,
    accepted)).  The ICP target is the map session's static map at 0.4 m."""
    T, fit, its, exs = register_session(xyzi, offsets, poses, oracle.voxel(map_static, 0.4), lidar2base, order, pose_offset)
    acc = fit < 1.0
    parts = split_session_refined(xyzi, offsets, poses, inv_poses, map_static, criterion, k, thr, T, acc, lidar2base, base2lidar, order,
                                  pose_offset)
    return parts, (T, fit, its, exs, acc)
