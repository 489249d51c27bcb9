"""CPU restatement of LT-map change composition and map rollback (DESIGN.md §5.3), the yardstick of ltr_knn_split_per_keyframe and of
ltrh_compose_changes / ltrh_rollback.  A scan set is a list of (n_k, 4) float32 arrays, one per keyframe, in that keyframe's frame.

  A (-) B   the points of A, in order, whose mean of the k smallest squared distances to B is not < thr (ltr_knn_split_cloud's rule:
            FLANN's L2_Simple in f32, summed ascending in double, float(sum) / float(k)); all n < k points of a small B count; empty B keeps A
  X ++ Y    concatenation, X first
  V(.)      octreeDownsampling(., 0.05) per keyframe
"""
import numpy as np

import oracle

LEAF = 0.05


def far_mask(a, b, k, thr, brute=False):
    """1 = far for every point of a against b."""
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
    b = np.ascontiguousarray(b, np.float32).reshape(-1, 4)
    if len(b) == 0:
        return np.ones(len(a), bool)
    if len(a) == 0:
        return np.zeros(0, bool)
    d = oracle.knn_dists(a, b, k, brute=brute)       # ascending; +inf beyond len(b)
    s = np.zeros(len(a), np.float64)
    for j in range(min(k, len(b))):
        s = s + d[:, j].astype(np.float64)
    avg = s.astype(np.float32) / np.float32(k)
    return ~(np.abs(avg) < np.float32(thr))


def minus(a, b, k, thr, brute=False):
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 4)
    return a[far_mask(a, b, k, thr, brute)]


def set_minus(A, B, k, thr):
    return [minus(a, b, k, thr) for a, b in zip(A, B)]


def concat(X, Y):
    return [np.concatenate([np.asarray(x, np.float32).reshape(-1, 4), np.asarray(y, np.float32).reshape(-1, 4)]) for x, y in zip(X, Y)]


def V(X):
    return [oracle.voxel(np.asarray(x, np.float32).reshape(-1, 4), LEAF) for x in X]


def compose(deltas, i, j, k, thr):
    """(PD, ND) over the generations [i, j) of deltas = [(PD_g, ND_g), ...]."""
    assert 0 <= i < j <= len(deltas)
    pd, nd = deltas[i]
    for g in range(i + 1, j):
        pdg, ndg = deltas[g]
        nd, pd = V(concat(set_minus(nd, pdg, k, thr), set_minus(ndg, pd, k, thr))), V(concat(set_minus(pd, ndg, k, thr), set_minus(pdg, nd, k, thr)))
    return pd, nd


def rollback(live, deltas, i, k, thr):
    """The scans as of generation i from the live scans after len(deltas) generations."""
    T = len(deltas)
    assert 0 <= i <= T
    if i == T:
        return [np.asarray(x, np.float32).reshape(-1, 4) for x in live]
    pd, nd = compose(deltas, i, T, k, thr)
    return V(concat(set_minus(live, pd, k, thr), nd))


def merged_map(scans, poses, leaf=LEAF, lidar2base=oracle.IDENTITY, order=0):
    """mergeAndDownsample(scans, leaf): every keyframe moved by lidar2base, then by its pose, in the given transform order, concatenated,
    voxelised.  An identity lidar2base is skipped, as the library skips it (ltr_merge_scans_global passes no extrinsic then); applying it
    would not be a no-op for -0.0 coordinates."""
    ident = np.array_equal(np.asarray(lidar2base, np.float64), np.eye(4))
    parts = []
    for s, p in zip(scans, poses):
        s = np.asarray(s, np.float32).reshape(-1, 4)
        parts.append(oracle.transform(s if ident else oracle.transform(s, lidar2base, order), p, order))
    return oracle.voxel(np.concatenate(parts) if parts else np.zeros((0, 4), np.float32), leaf)


def split_sets(pts, off):
    return [pts[off[k]:off[k + 1]] for k in range(len(off) - 1)]


def pack(X):
    """(points, offsets) of a list of per-keyframe arrays."""
    X = [np.asarray(x, np.float32).reshape(-1, 4) for x in X]
    off = np.concatenate([[0], np.cumsum([len(x) for x in X])]).astype(np.int64)
    return (np.concatenate(X) if X else np.zeros((0, 4), np.float32)), off
