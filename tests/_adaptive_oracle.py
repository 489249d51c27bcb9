"""CPU restatement of the remove / revert / ND / PD pass with the range-adaptive discrepancy threshold (test infrastructure, not
product code).

calcDescrepancyAndParseDynamicPointIdx (ltremovert/src/Removerter.cpp:381-413) with its commented-out line 396 in place of line 398:
a pixel's threshold is fl(c * s), s the keyframe's scan range at the pixel (10000 without a return).  Built from the oracle's
primitives only -- scan2RangeImg (oracle.scan2rimg), the two-step map transform (oracle.transform) and map2RangeImg (oracle.map2rimg:
minimum range, lowest index on ties, 10000 / index 0 where no map point falls) -- so that the threshold rule is the only new part, and
that rule is restated here in numpy float32.
"""
import numpy as np

import oracle

F32 = np.float32
VALID_DIFF_UPPER_BOUND = F32(200.0)   # utility.h:94


def pixel_flags(scan_rimg, map_rimg, mode, coeff):
    """Removerter.cpp:388-410 with line 396: per pixel, diff = scan - map (HD / revert / PD, :572 / :459) or map - scan (ND, :516),
    t = fl(coeff * scan), flagged iff diff < 200 && diff > t.  Every operation is one float32 operation."""
    s = np.asarray(scan_rimg, F32)
    m = np.asarray(map_rimg, F32)
    diff = (m - s) if mode == oracle.MODE_ND else (s - m)
    t = F32(coeff) * s
    return (diff < VALID_DIFF_UPPER_BOUND) & (diff > t)


def _is_identity(m):
    return np.array_equal(np.asarray(m, np.float64), np.eye(4))


def remove_pass(map_xyzi, scans_xyzi, offsets, inv_poses, mode, alpha, coeff, vfov=50.0, hfov=360.0, lidar2base=oracle.IDENTITY, order=0):
    """flags (N,) uint8, 1 = dynamic: the union over the keyframes of the flagged pixels' winners (Removerter.cpp:542-593, 485-540,
    429-482)."""
    m = np.ascontiguousarray(map_xyzi, F32)
    s = np.ascontiguousarray(scans_xyzi, F32)
    rows, cols = oracle.reset_rimg_size(alpha, vfov, hfov)
    base2lidar = None if _is_identity(lidar2base) else oracle.inverse4x4(lidar2base)
    flags = np.zeros(len(m), np.uint8)
    for k in range(len(offsets) - 1):
        srimg = oracle.scan2rimg(s[offsets[k]:offsets[k + 1]], rows, cols, vfov, hfov)
        if len(m) == 0:
            continue
        local = oracle.transform(m, inv_poses[k], order)
        if base2lidar is not None:
            local = oracle.transform(local, base2lidar, order)
        mrimg, idx = oracle.map2rimg(local, rows, cols, vfov, hfov)
        flags[idx[pixel_flags(srimg, mrimg, mode, coeff)]] = 1
    return flags
