"""Edge cases of the C-ABI: empty and ragged inputs, inputs on which the reference has undefined behaviour, error codes."""
import numpy as np
import pytest

import oracle
import lt_mapper_b200 as ltr

pytestmark = pytest.mark.gpu
I4 = np.eye(4)[None]


@pytest.fixture(scope="module")
def ctx():
    c = ltr.Context()
    yield c
    c.close()


def test_empty_inputs(ctx):
    e = np.zeros((0, 4), np.float32)
    c = ctx.cloud_upload(e)
    assert ctx.cloud_size(c) == 0 and ctx.cloud_download(c).shape == (0, 4)
    assert ctx.cloud_size(ctx.voxel_centroid(c, 0.05)) == 0                       # empty in -> empty out (PCL: empty octree)
    s, d = ctx.apply_partition(c)                                                 # N == 0: linspace yields an empty index set
    assert ctx.cloud_size(s) == 0 and ctx.cloud_size(d) == 0
    ss = ctx.scanset_upload(e, [0, 0, 0])                                         # two keyframes without points
    ps = ctx.poses_upload(np.repeat(I4, 2, 0), np.repeat(I4, 2, 0))
    assert ctx.cloud_size(ctx.merge_scans_global(ss, ps)) == 0
    m = ctx.cloud_upload(np.array([[5, 0, 0, 1], [0, 5, 0, 2], [0, 0, 5, 3]], np.float32))
    assert ctx.remove_pass(m, ss, ps, ltr.MODE_HD, 2.5) == 0                      # no scan returns -> nothing can be flagged
    assert ctx.remove_pass(c, ss, ps, ltr.MODE_ND, 2.5) == 0                      # empty map
    vis = ctx.parse_projected(c, ps, 0, 2, 3.0)
    assert ctx.scanset_info(vis) == (2, 0)
    co, di = ctx.knn_diff(ss, ps, m, 1, 0.04)
    assert ctx.scanset_info(co) == (2, 0) and ctx.scanset_info(di) == (2, 0)
    assert ctx.scanset_info(ctx.preclean(ss, 2.5)) == (2, 0)


def test_ragged_keyframes(ctx):
    """Keyframes of very different sizes, including empty ones in the middle, keep per-keyframe order and offsets."""
    rng = np.random.default_rng(3)
    sizes = [0, 1, 1000, 0, 37, 5000, 0]
    pts = rng.uniform(-30, 30, (sum(sizes), 4)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)])
    K = len(sizes)
    poses = np.repeat(I4, K, 0).copy()
    poses[:, 0, 3] = np.arange(K)
    inv = oracle.inverse_poses(poses)
    ss = ctx.scanset_upload(pts, off)
    ps = ctx.poses_upload(poses, inv)
    target = rng.uniform(-30, 30, (20000, 4)).astype(np.float32)
    th = ctx.cloud_upload(target)
    co, di = ctx.knn_diff(ss, ps, th, 2, 1.0)
    cp, coff = ctx.scanset_download(co)
    dp, doff = ctx.scanset_download(di)
    for k in range(K):
        lab, eco, edi = oracle.knn_partition(pts[off[k]:off[k + 1]], poses[k], inv[k], target, 2, 1.0)
        assert np.array_equal(cp[coff[k]:coff[k + 1]].view(np.uint32), eco.view(np.uint32))
        assert np.array_equal(dp[doff[k]:doff[k + 1]].view(np.uint32), edi.view(np.uint32))
    pre = ctx.preclean(ss, 25.0)
    pp, poff = ctx.scanset_download(pre)
    for k in range(K):
        s = pts[off[k]:off[k + 1]]
        r = np.sqrt((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1] + s[:, 2] * s[:, 2]).astype(np.float32), dtype=np.float32)
        keep = ~((r < 25.0) & (s[:, 2] < 0.5) & (-0.5 < s[:, 2]))                # Session.cpp:522-526
        assert np.array_equal(pp[poff[k]:poff[k + 1]], s[keep])
    m = oracle.voxel(target, 0.5)
    mh = ctx.cloud_upload(m)
    n = ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)
    exp = oracle.remove_pass(m, pts, off, inv, oracle.MODE_HD, 2.5)
    assert n == int(exp.sum()) and np.array_equal(ctx.flags_download(mh), exp)


def test_reference_undefined_behaviour_is_rejected(ctx):
    # getStaticIdxFromDynamicIdx: linspace<int>(0, N, N) divides by N-1 == 0 for N == 1 and indexes out of range for N == 2
    for n in (1, 2):
        m = ctx.cloud_upload(np.ones((n, 4), np.float32))
        with pytest.raises(ltr.LtrError) as e:
            ctx.apply_partition(m)
        assert e.value.code == -3
    # kNN against an empty target (PCL asserts on an empty tree)
    ss = ctx.scanset_upload(np.ones((5, 4), np.float32), [0, 5])
    ps = ctx.poses_upload(I4, I4)
    with pytest.raises(ltr.LtrError) as e:
        ctx.knn_diff(ss, ps, ctx.cloud_upload(np.zeros((0, 4), np.float32)), 2, 0.01)
    assert e.value.code == -3


@pytest.mark.parametrize("n_target,k,thr", [(1, 2, 0.01), (1, 2, 1.0), (2, 3, 0.5), (3, 5, 2.0)])
def test_knn_target_smaller_than_k(ctx, n_target, k, thr):
    """Fewer target points than k: PCL's nearestKSearch returns all of them and the reference still divides their sum by k
    (Session.cpp:470-471, 592-594) -- e.g. a strong-ND map of one point in removeWeakNDMapPointsHavingStrongNDInNear.  The device path
    must give the oracle's partition, not an error."""
    rng = np.random.default_rng(5 + n_target)
    tgt = np.zeros((n_target, 4), np.float32); tgt[:, :3] = rng.uniform(-1, 1, (n_target, 3))
    q = np.zeros((4000, 4), np.float32); q[:, :3] = rng.uniform(-2, 2, (4000, 3)); q[:, 3] = np.arange(4000)
    q[:50, :3] = tgt[0, :3] + rng.normal(0, 0.02, (50, 3)).astype(np.float32)
    ss = ctx.scanset_upload(q, [0, len(q)])
    ps = ctx.poses_upload(I4, I4)
    th = ctx.cloud_upload(tgt)
    co, di = ctx.knn_diff(ss, ps, th, k, thr)
    lab, eco, edi = oracle.knn_partition(q, I4[0] if I4.ndim == 3 else I4, I4[0] if I4.ndim == 3 else I4, tgt, k, thr)
    cp, _ = ctx.scanset_download(co); dp, _ = ctx.scanset_download(di)
    assert 0 < len(edi) < len(q)
    assert np.array_equal(cp.view(np.uint32), eco.view(np.uint32)) and np.array_equal(dp.view(np.uint32), edi.view(np.uint32))
    near, far = ctx.knn_split_cloud(ctx.cloud_upload(q), th, k, thr)
    assert np.array_equal(ctx.cloud_download(near), q[lab == 0]) and np.array_equal(ctx.cloud_download(far), q[lab == 1])


def test_argument_errors(ctx):
    m = ctx.cloud_upload(np.ones((10, 4), np.float32))
    ss = ctx.scanset_upload(np.ones((5, 4), np.float32), [0, 5])
    ps2 = ctx.poses_upload(np.repeat(I4, 2, 0), np.repeat(I4, 2, 0))
    with pytest.raises(ltr.LtrError) as e:                                        # pose count != scan count (Session.cpp:117 assert)
        ctx.remove_pass(m, ss, ps2, ltr.MODE_HD, 2.5)
    assert e.value.code == -1
    with pytest.raises(ltr.LtrError):
        ctx.cloud_size(12345)
    with pytest.raises(ltr.LtrError):
        ctx.remove_pass(m, ss, ctx.poses_upload(I4, I4), 7, 2.5)                   # unknown mode
    with pytest.raises(ltr.LtrError):
        ctx.scanset_upload(np.ones((5, 4), np.float32), [0, 7, 5])                 # decreasing offsets
    with pytest.raises(ltr.LtrError):
        ctx.voxel_centroid(m, -1.0)
    ctx.cloud_free(m)
    with pytest.raises(ltr.LtrError):                                             # use after free
        ctx.cloud_size(m)


def test_degenerate_geometry_goes_through_the_exact_path(ctx):
    """Points at the sensor origin, on the vertical axis and on the azimuth seam (fast path must defer to the exact one)."""
    m = np.array([[0, 0, 0, 1], [0, 0, 3, 2], [0, 0, -3, 3], [-5, 0.0, 0, 4], [-5, -1e-7, 0, 5], [-5, 1e-7, 0, 6], [1e-20, 1e-20, 1e-20, 7],
                  [4, 0, 0, 8], [1e4, 0, 0, 9]], np.float32)
    scan = np.array([[6, 0, 0, 0], [-7, 0, 0, 0], [0, 0, 8, 0], [0, 0, -8, 0], [-7, -1e-6, 0, 0]], np.float32)
    exp = oracle.remove_pass(m, scan, [0, len(scan)], I4, oracle.MODE_HD, 2.5)
    mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(scan, [0, len(scan)]); ps = ctx.poses_upload(I4, I4)
    for mode in (ltr.MODE_HD, ltr.MODE_ND, ltr.MODE_PD):
        e = oracle.remove_pass(m, scan, [0, len(scan)], I4, mode, 2.5)
        ctx.remove_pass(mh, ss, ps, mode, 2.5)
        assert np.array_equal(ctx.flags_download(mh), e), mode
    pts, off = ctx.scanset_download(ctx.parse_projected(mh, ps, 0, 1, 3.0))
    ep, _ = oracle.parse_projected(m, I4[0], 3.0)
    assert np.array_equal(pts.view(np.uint32), ep.view(np.uint32))
    assert exp.sum() > 0


def test_error_paths_release_their_scratch_memory(ctx):
    """Calls that fail half-way (non-finite coordinates in the voxeliser, kNN against too few points, bad arguments to a pass) and
    calls that succeed leave the allocator's live byte count exactly where the handles they created account for it."""
    good = np.random.default_rng(0).uniform(-5, 5, (200000, 4)).astype(np.float32)
    bad = good.copy(); bad[1234, 1] = np.nan
    hg, hb = ctx.cloud_upload(good), ctx.cloud_upload(bad)
    ss = ctx.scanset_upload(good[:1000], [0, 400, 1000])
    ps = ctx.poses_upload(np.stack([I4, I4]), np.stack([I4, I4]))
    tiny = ctx.cloud_upload(good[:0])                          # an empty kNN target is rejected (PCL asserts on an empty tree)
    ss_bad = ctx.scanset_upload(bad[:2000], [0, 1000, 2000])   # the non-finite point lies in the second keyframe
    base = ctx.memory_stats()[0]
    for _ in range(3):
        with pytest.raises(ltr.LtrError):
            ctx.voxel_centroid(hb, 0.1)                       # fails after the output cloud, keys and scratch were allocated
        with pytest.raises(ltr.LtrError) as e:
            ctx.voxel_centroid_per_keyframe(ss_bad, 0.1)      # fails after the first keyframe was voxelised into the scratch cloud
        assert e.value.code == -3
        with pytest.raises(ltr.LtrError):
            ctx.knn_diff(ss, ps, tiny, 2, 0.01)
        with pytest.raises(ltr.LtrError):
            ctx.remove_pass(hg, ss, ps, 7, 2.5)                # unknown mode
        assert ctx.memory_stats()[0] == base
    ctx.remove_pass(hg, ss, ps, ltr.MODE_HD, 2.5)              # first pass on hg allocates its flag array (stays with the handle)
    ctx.cloud_free(ctx.voxel_centroid(hg, 0.1))
    before = ctx.memory_stats()[0]
    ctx.remove_pass(hg, ss, ps, ltr.MODE_HD, 2.5)
    ctx.cloud_free(ctx.voxel_centroid(hg, 0.1))
    assert ctx.memory_stats()[0] == before                     # steady state: scratch goes back to the cache


def test_randomised_small_passes_match_the_oracle():
    """Many tiny random scenes (not geometrically consistent; coarse images so pixels collide, duplicated points so ranges tie, signed zeros,
    points on the sensor axis) through every pass variant and the visible-point extraction: flags / points equal the oracle's (whose
    behaviour on exactly such inputs is pinned against the compiled reference by the property tests in tests/test_ref_pin.py)."""
    rng = np.random.default_rng(2024)
    with ltr.Context() as ctx, ltr.Context(fast_path=False) as ctx_exact:
        for case in range(60):
            n = int(rng.integers(3, 500))
            m = np.concatenate([rng.normal(0, 15, (n, 3)), rng.uniform(0, 1, (n, 1))], 1).astype(np.float32)
            if case % 3 == 0:
                m = np.concatenate([m, m[: n // 2]])                                   # exact range ties
            if case % 5 == 0:
                m[: min(4, len(m)), :3] = [[0.0, 0.0, 0.0], [-0.0, 0.0, 0.0], [0.0, 0.0, 2.0], [0.0, -0.0, -3.0]][: min(4, len(m))]
            K = int(rng.integers(1, 4))
            scans = []
            for _ in range(K):
                ns = int(rng.integers(0, 300))
                scans.append(np.concatenate([rng.normal(0, 15, (ns, 3)), np.zeros((ns, 1))], 1).astype(np.float32))
            xyzi = np.concatenate(scans) if sum(map(len, scans)) else np.zeros((0, 4), np.float32)
            off = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
            poses = np.stack([np.eye(4) for _ in range(K)])
            for k in range(K):
                a = rng.uniform(-np.pi, np.pi)
                poses[k][:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
                poses[k][:3, 3] = rng.normal(0, 5, 3)
            inv = oracle.inverse_poses(poses)
            alpha = [0.2, 0.5, 1.0, 2.5][case % 4]
            for c in (ctx, ctx_exact):
                mh = c.cloud_upload(m); ss = c.scanset_upload(xyzi, off); ps = c.poses_upload(poses, inv)
                for mode, omode in ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_ND, oracle.MODE_ND), (ltr.MODE_PD, oracle.MODE_PD)):
                    exp = oracle.remove_pass(m, xyzi, off, inv, omode, alpha, 0.1)
                    c.remove_pass(mh, ss, ps, mode, alpha)
                    assert np.array_equal(c.flags_download(mh), exp), (case, mode, c is ctx)
                pts, po = c.scanset_download(c.parse_projected(mh, ps, 0, K, alpha))
                for k in range(K):
                    e, _ = oracle.parse_projected(m, inv[k], alpha)
                    assert np.array_equal(pts[po[k]:po[k + 1]].view(np.uint32), e.view(np.uint32)), (case, k, c is ctx)
                c.cloud_free(mh)
