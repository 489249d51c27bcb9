"""ICP refinement on the GPU (ltr_icp_refine, ltr_knn_diff_refined; icp.cu) against the CPU restatement (tests/_icp_oracle.py), bit for bit
in the final transforms, fitness, iterations, exit reasons and both scan sets."""
import numpy as np
import pytest

import oracle
import _icp_oracle as io

pytestmark = pytest.mark.gpu


def _rot(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    R = np.eye(4)
    R[i, i] = c; R[j, j] = c; R[i, j] = -s; R[j, i] = s
    return R


def _perturb(poses, trans=0.3, deg=1.0):
    E = _rot(2, deg) @ _rot(0, deg / 3)
    E[:3, 3] = np.array([1.0, -0.6, 0.2]) * trans
    return np.stack([p @ E for p in poses])


def _per_kf(pts, off):
    return [pts[off[j]:off[j + 1]] for j in range(len(off) - 1)]


def _same(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _run(ctx, xyzi, offsets, poses, target_down, target, k=2, thr=0.01, pose_offset=0, b2l=oracle.IDENTITY, **params):
    """Device refinement + partition, checked against the restatement; returns (accepted mask, fitness, exits)."""
    inv = oracle.inverse_poses(poses)
    ss = ctx.scanset_upload(xyzi, offsets)
    ps = ctx.poses_upload(poses, inv)
    td = ctx.cloud_upload(target_down)
    th = ctx.cloud_upload(target)
    T, fit, it, ex = ctx.icp_refine(ss, ps, td, pose_offset=pose_offset, **params)
    eT, efit, eit, eex = io.refine_session(xyzi, offsets, poses, target_down, b2l, pose_offset=pose_offset, **params)
    assert np.array_equal(it, eit) and np.array_equal(ex, eex), (it, eit, ex, eex)
    assert _same(T, eT), np.abs(T - eT).max()
    assert np.array_equal(fit.view(np.uint64), efit.view(np.uint64)), (fit, efit)
    acc = fit < 1.0
    co, di = ctx.knn_diff_refined(ss, ps, th, k, thr, T, acc, pose_offset=pose_offset)
    pco, pdi = ctx.knn_diff(ss, ps, th, k, thr, pose_offset=pose_offset)
    exp = io.knn_diff_refined(xyzi, offsets, poses, inv, target, k, thr, eT, acc, b2l, pose_offset=pose_offset)
    for part, (h, hp) in enumerate(((co, pco), (di, pdi))):
        got = _per_kf(*ctx.scanset_download(h))
        plain = _per_kf(*ctx.scanset_download(hp))
        for kf in range(len(offsets) - 1):
            assert _same(got[kf], exp[part][kf]), (part, kf)
            if not acc[kf]:
                assert _same(got[kf], plain[kf]), ("a keyframe that is not accepted must equal ltr_knn_diff", part, kf)
        ctx.scanset_free(h)
        ctx.scanset_free(hp)
    ctx.scanset_free(ss)
    ctx.poses_free(ps)
    ctx.cloud_free(td)
    ctx.cloud_free(th)
    return acc, fit, ex


@pytest.mark.parametrize("perturbed", [False, True])
def test_sessions_match_the_restatement(small_pair, small_maps, perturbed):
    """Central keyframes against the query session's map (Step 2's pairing), with the synthetic poses and with a known pose error."""
    import lt_mapper_b200 as ltr
    c = small_pair[0].subset(0, 4)
    poses = _perturb(c.poses) if perturbed else c.poses
    m = small_maps[1]
    md = oracle.voxel(m, 0.4)
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        acc, fit, ex = _run(ctx, c.xyzi, c.offsets, poses, md, m)
        assert acc.any()
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0


def test_edge_keyframes_lattice_ties_chunks_and_iteration_cap(small_pair, small_maps, monkeypatch):
    """Empty, 1- and 2-point keyframes (fewer than 3 correspondences), a keyframe far from every map point (no pair within 150 m), a
    keyframe that half-overlaps the map (it registers, moves, and still has fitness >= 1.0: not accepted), a lattice keyframe against a
    lattice target half a step away (every nearest neighbour a tie), launches of one keyframe, a lowered iteration cap (exit 1), and the
    two MSE tests with the increment test off (exit 3 when both hold, exit 4 when only the relative one does)."""
    import lt_mapper_b200 as ltr
    c = small_pair[0].subset(0, 2)
    ax = np.arange(-6, 7, dtype=np.float32) * 0.5
    g = np.stack(np.meshgrid(ax, ax, ax[:5], indexing="ij"), -1).reshape(-1, 3)
    lat = np.concatenate([g, np.ones((len(g), 1))], 1).astype(np.float32)
    far = np.random.default_rng(4).uniform(-50, 50, (400, 4)).astype(np.float32)   # 500 m from the map: no pair within 150 m
    far[:, 0] += 500.0
    lifted = c.scan(1).copy()
    lifted[:, 2] += 8.0                                # the scan and a copy 8 m above it: half of it can never fit
    half = np.concatenate([c.scan(1), lifted])
    scans = [np.zeros((0, 4), np.float32), c.scan(0)[:1], c.scan(0)[:2], c.scan(1), far, lat, half]
    xyzi = np.concatenate(scans)
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
    pert = _perturb(c.poses[1:2])[0]
    poses = np.stack([c.poses[0], c.poses[0], c.poses[0], pert, c.poses[0], np.eye(4), pert])
    tlat = np.concatenate([(g + np.float32(0.25)), np.zeros((len(g), 1))], 1).astype(np.float32)
    target = np.concatenate([small_maps[0], tlat, tlat]).astype(np.float32)   # the lattice twice: ties between copies too
    md = oracle.voxel(small_maps[0], 0.4)
    md = np.concatenate([md, tlat, tlat[::-1]]).astype(np.float32)
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        acc, fit, ex = _run(ctx, xyzi, offsets, poses, md, target)
        assert list(ex[:3]) == [io.NO_CORRESPONDENCES] * 3 and fit[0] == io.DBL_MAX
        assert fit[4] >= 1.0 and not acc[4] and acc[3]
        # the rejected keyframe 6 did move: honouring the mask is what keeps ltr_knn_diff's bytes (checked in _run)
        ss = ctx.scanset_upload(xyzi, offsets)
        ps = ctx.poses_upload(poses, oracle.inverse_poses(poses))
        td, th = ctx.cloud_upload(md), ctx.cloud_upload(target)
        T, fit, it, ex = ctx.icp_refine(ss, ps, td)
        assert fit[6] >= 1.0 and it[6] > 1 and np.abs(T[6] - np.eye(4, dtype=np.float32)).max() > 0.1
        def diff_part(pair):
            out = _per_kf(*ctx.scanset_download(pair[1]))
            for h in pair:
                ctx.scanset_free(h)
            return out
        forced = diff_part(ctx.knn_diff_refined(ss, ps, th, 2, 0.01, T, np.ones(len(T), bool)))
        masked = diff_part(ctx.knn_diff_refined(ss, ps, th, 2, 0.01, T, fit < 1.0))
        plain = diff_part(ctx.knn_diff(ss, ps, th, 2, 0.01))
        assert _same(masked[6], plain[6]) and not _same(forced[6], plain[6])
        ctx.scanset_free(ss)
        ctx.poses_free(ps)
        ctx.cloud_free(td)
        ctx.cloud_free(th)
        for chunk in ("1", "700"):
            monkeypatch.setenv("LTR_ICP_CHUNK_POINTS", chunk)
            _run(ctx, xyzi, offsets, poses, md, target)
        monkeypatch.delenv("LTR_ICP_CHUNK_POINTS")
        _, _, ex = _run(ctx, xyzi, offsets, poses, md, target, max_iterations=2)
        assert ex[3] == io.ITERATIONS and ex[5] in (io.ITERATIONS, io.TRANSFORM)
        _, _, ex = _run(ctx, xyzi, offsets, poses, md, target, transformation_epsilon=0.0, mse_threshold_absolute=1e-3)
        assert ex[3] == io.ABS_MSE
        _, _, ex = _run(ctx, xyzi, offsets, poses, md, target, transformation_epsilon=0.0, euclidean_fitness_epsilon=1e-2)
        assert ex[3] == io.REL_MSE
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0


def test_non_identity_extrinsic_and_pose_offset(small_pair, small_maps):
    import lt_mapper_b200 as ltr
    a = 0.05
    l2b = np.array([[np.cos(a), 0, np.sin(a), 0.3], [0, 1, 0, -0.02], [-np.sin(a), 0, np.cos(a), 1.1], [0, 0, 0, 1]])
    b2l = oracle.inverse4x4(l2b)
    full = small_pair[0]
    s = full.subset(2, 5)
    poses = _perturb(full.poses, 0.2, 0.5)
    md = oracle.voxel(small_maps[1], 0.4)
    with ltr.Context(device=0, lidar2base=l2b, base2lidar=b2l) as ctx:
        _run(ctx, s.xyzi, s.offsets, poses, md, small_maps[1], pose_offset=2, b2l=b2l)


def test_rejections():
    import lt_mapper_b200 as ltr
    scan = np.array([[1, 2, 3, 0], [4, 5, 6, 0], [7, 1, 2, 0]], np.float32)
    off = np.array([0, 3], np.int64)
    pose = np.eye(4)[None]
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        ss = ctx.scanset_upload(scan, off)
        ps = ctx.poses_upload(pose, pose)
        empty = ctx.cloud_upload(np.zeros((0, 4), np.float32))
        bad = ctx.cloud_upload(np.array([[0, 0, 0, 0], [np.nan, 0, 0, 0], [1, 1, 1, 0]], np.float32))
        good = ctx.cloud_upload(scan)
        bad_scan = ctx.scanset_upload(np.array([[np.inf, 0, 0, 0]], np.float32), np.array([0, 1], np.int64))
        for args in ((ss, ps, empty), (ss, ps, bad), (bad_scan, ps, good)):
            with pytest.raises(ltr.LtrError):
                ctx.icp_refine(*args)
        with pytest.raises(ltr.LtrError):
            ctx.icp_refine(ss, ps, good, max_iterations=0)
        with pytest.raises(ltr.LtrError):
            ctx.icp_refine(ss, ps, good, pose_offset=1)
        with pytest.raises(ltr.LtrError):
            ctx.knn_diff_refined(ss, ps, empty, 2, 0.1, np.eye(4, dtype=np.float32)[None], [1])
        for h in (empty, bad, good):
            ctx.cloud_free(h)
        for h in (ss, bad_scan):
            ctx.scanset_free(h)
        ctx.poses_free(ps)
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0
