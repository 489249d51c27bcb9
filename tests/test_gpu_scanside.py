"""Scan-side removal on the GPU (ltr_scanside_split, scanside.cu) against the CPU restatement (tests/_scanside_oracle.py), byte for byte."""
import numpy as np
import pytest

import oracle
import _scanside_oracle as so

pytestmark = pytest.mark.gpu
CRITERIA = {"map": so.MAP, "scan_minus_map": so.SCAN_MINUS_MAP}


def _inv(poses):
    return np.stack([oracle.inverse4x4(p) for p in poses]) if len(poses) else np.zeros((0, 4, 4))


def _device(ctx, xyzi, offsets, poses, map_xyzi, criterion, k, thr):
    import lt_mapper_b200 as ltr  # noqa: F401
    ss = ctx.scanset_upload(xyzi, offsets)
    ps = ctx.poses_upload(poses, _inv(poses))
    mh = ctx.cloud_upload(map_xyzi)
    st, dy = ctx.scanside_split(ss, ps, mh, criterion, k, thr)
    out = []
    for h in (st, dy):
        pts, off = ctx.scanset_download(h)
        out.append([pts[off[j]:off[j + 1]] for j in range(len(off) - 1)])
        ctx.scanset_free(h)
    for h in (ss,):
        ctx.scanset_free(h)
    ctx.poses_free(ps)
    ctx.cloud_free(mh)
    return out


def _assert_equal(dev, exp):
    for part in range(2):
        assert len(dev[part]) == len(exp[part])
        for kf, (a, b) in enumerate(zip(dev[part], exp[part])):
            assert a.shape == b.shape, f"part {part} keyframe {kf}: {a.shape} vs {b.shape}"
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"part {part} keyframe {kf} differs"


def _check(ctx, xyzi, offsets, poses, map_xyzi, criterion, k, thr, l2b=oracle.IDENTITY):
    dev = _device(ctx, xyzi, offsets, poses, map_xyzi, criterion, k, thr)
    exp = so.split_session(xyzi, offsets, poses, _inv(poses), map_xyzi, criterion, k, thr, l2b, oracle.inverse4x4(l2b) if l2b is not oracle.IDENTITY else oracle.IDENTITY)
    _assert_equal(dev, exp)
    return dev


@pytest.mark.parametrize("criterion", list(CRITERIA))
@pytest.mark.parametrize("pair", ["CC", "QQ", "CQ", "QC"])
def test_session_pairs_match_the_oracle(small_pair, small_maps, criterion, pair):
    """(map session, scan session) = (C,C), (Q,Q): self-cleaning; (C,Q), (Q,C): scan-level positive / negative differences."""
    import lt_mapper_b200 as ltr
    m = small_maps["CQ".index(pair[0])]
    s = small_pair["CQ".index(pair[1])]
    with ltr.Context(device=0) as ctx:
        for k, thr in ((3, 0.1), (1, 0.01), (16, 0.5)):
            dev = _check(ctx, s.xyzi, s.offsets, s.poses, m, CRITERIA[criterion], k, thr)
            n_st, n_dy = sum(len(a) for a in dev[0]), sum(len(a) for a in dev[1])
            assert n_st + n_dy == len(s.xyzi)


def _edge_session(rng):
    """Keyframes: empty, fewer than k points, duplicates, a rotated 0.25 m lattice, isolated points tens of metres apart."""
    scans = [np.zeros((0, 4), np.float32), np.array([[1, 2, 3, 7], [1.5, 2, 3, 8]], np.float32)]
    d = rng.normal(0, 2, (300, 4)).astype(np.float32)
    d[100:200] = d[:100]
    scans.append(d)
    g = np.stack(np.meshgrid(np.arange(-4, 5) * 0.25, np.arange(-4, 5) * 0.25, np.arange(-2, 3) * 0.25, indexing="ij"), -1).reshape(-1, 3)
    scans.append(np.concatenate([g, np.ones((len(g), 1))], 1).astype(np.float32))
    far = np.concatenate([rng.uniform(-1, 1, (40, 3)) * 60.0, np.zeros((40, 1))], 1).astype(np.float32)
    scans.append(far)
    offsets = np.concatenate([[0], np.cumsum([len(x) for x in scans])]).astype(np.int64)
    poses = []
    for j in range(len(scans)):
        a = 0.2 * j
        poses.append(np.array([[np.cos(a), -np.sin(a), 0, 0.37 * j], [np.sin(a), np.cos(a), 0, -0.11 * j], [0, 0, 1, 0.05 * j], [0, 0, 0, 1]]))
    return np.concatenate(scans), offsets, np.stack(poses)


@pytest.mark.parametrize("criterion", list(CRITERIA))
def test_edge_cases(criterion, monkeypatch):
    import lt_mapper_b200 as ltr
    rng = np.random.default_rng(3)
    xyzi, offsets, poses = _edge_session(rng)
    map_big = np.concatenate([rng.normal(0, 3, (2000, 4)), rng.uniform(-70, 70, (50, 4))]).astype(np.float32)
    map_big[:, 3] = 0
    map_big[10:20] = map_big[:10]
    crit = CRITERIA[criterion]
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        for k in (1, 2, 3, 5, 16):
            _check(ctx, xyzi, offsets, poses, map_big, crit, k, 0.05)
            _check(ctx, xyzi, offsets, poses, map_big[:max(1, k - 1)], crit, k, 0.05)       # a map with fewer than k points
        st = ctx.scanside_stats()
        assert st[0] == len(xyzi)
        if crit == so.SCAN_MINUS_MAP:
            assert st[2] > 0, "the isolated points must reach the expanding pass"
        for chunk in ("1", "300", "700"):                                                     # launch splitting
            monkeypatch.setenv("LTR_SCANSIDE_CHUNK_POINTS", chunk)
            _check(ctx, xyzi, offsets, poses, map_big, crit, 3, 0.05)
        monkeypatch.delenv("LTR_SCANSIDE_CHUNK_POINTS")
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0


@pytest.mark.parametrize("criterion", list(CRITERIA))
def test_non_identity_extrinsic(small_pair, small_maps, criterion):
    import lt_mapper_b200 as ltr
    a = 0.05
    l2b = np.array([[np.cos(a), 0, np.sin(a), 0.3], [0, 1, 0, -0.02], [-np.sin(a), 0, np.cos(a), 1.1], [0, 0, 0, 1]])
    b2l = oracle.inverse4x4(l2b)
    s = small_pair[0].subset(0, 3)
    with ltr.Context(device=0, lidar2base=l2b, base2lidar=b2l) as ctx:
        dev = _device(ctx, s.xyzi, s.offsets, s.poses, small_maps[0], CRITERIA[criterion], 3, 0.1)
    exp = so.split_session(s.xyzi, s.offsets, s.poses, _inv(s.poses), small_maps[0], CRITERIA[criterion], 3, 0.1, l2b, b2l)
    _assert_equal(dev, exp)


def test_rejections():
    import lt_mapper_b200 as ltr
    scan = np.array([[1, 2, 3, 0], [4, 5, 6, 0]], np.float32)
    off = np.array([0, 2], np.int64)
    pose = np.eye(4)[None]
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        ss = ctx.scanset_upload(scan, off)
        ps = ctx.poses_upload(pose, pose)
        for crit in (so.MAP, so.SCAN_MINUS_MAP):
            empty = ctx.cloud_upload(np.zeros((0, 4), np.float32))
            with pytest.raises(ltr.LtrError):
                ctx.scanside_split(ss, ps, empty, crit, 2, 0.1)
            bad = ctx.cloud_upload(np.array([[0, 0, 0, 0], [np.nan, 0, 0, 0], [1, 1, 1, 0]], np.float32))
            with pytest.raises(ltr.LtrError):
                ctx.scanside_split(ss, ps, bad, crit, 2, 0.1)
            bad_scan = ctx.scanset_upload(np.array([[np.inf, 0, 0, 0]], np.float32), np.array([0, 1], np.int64))
            good = ctx.cloud_upload(scan)
            with pytest.raises(ltr.LtrError):
                ctx.scanside_split(bad_scan, ps, good, crit, 2, 0.1)
            with pytest.raises(ltr.LtrError):
                ctx.scanside_split(ss, ps, good, crit, 17, 0.1)
            for h in (empty, bad, good):
                ctx.cloud_free(h)
            ctx.scanset_free(bad_scan)
        ctx.scanset_free(ss)
        ctx.poses_free(ps)
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0


@pytest.mark.parametrize("criterion", list(CRITERIA))
def test_points_exactly_on_cell_boundaries(criterion):
    """Identity pose, a lattice of 0.25 m steps (the finest cell side) starting at the box minimum: every global coordinate sits exactly on
    a cell face of both the own-scan grid and the map grid, where floor() decides the cell.  Duplicated lattice points and a sparser
    copy of the lattice as the map exercise ties at the k-th distance."""
    import lt_mapper_b200 as ltr
    ax = np.arange(-8, 9) * 0.25
    g = np.stack(np.meshgrid(ax, ax, ax[:9], indexing="ij"), -1).reshape(-1, 3)
    scan = np.concatenate([g, np.zeros((len(g), 1))], 1).astype(np.float32)
    scan = np.concatenate([scan, scan[::7]])
    for m in (scan[::3], scan[::2] + np.float32([0.25, 0, 0, 0])):
        with ltr.Context(device=0) as ctx:
            for k, thr in ((1, 0.01), (4, 0.02), (16, 0.05)):
                _check(ctx, scan, np.array([0, len(scan)], np.int64), np.eye(4)[None], m, CRITERIA[criterion], k, thr)


@pytest.mark.parametrize("criterion", list(CRITERIA))
def test_pose_offset(small_pair, small_maps, criterion):
    """Scans of keyframes 2..4 against a pose table of all keyframes, as a rank-local block indexes it."""
    import lt_mapper_b200 as ltr
    full = small_pair[1]
    s = full.subset(2, 5)
    inv = _inv(full.poses)
    with ltr.Context(device=0) as ctx:
        ss = ctx.scanset_upload(s.xyzi, s.offsets)
        ps = ctx.poses_upload(full.poses, inv)
        mh = ctx.cloud_upload(small_maps[0])
        st, dy = ctx.scanside_split(ss, ps, mh, CRITERIA[criterion], 3, 0.1, pose_offset=2)
        dev = []
        for h in (st, dy):
            pts, off = ctx.scanset_download(h)
            dev.append([pts[off[j]:off[j + 1]] for j in range(len(off) - 1)])
        with pytest.raises(ltr.LtrError):
            ctx.scanside_split(ss, ps, mh, CRITERIA[criterion], 3, 0.1, pose_offset=full.K - 2)
    exp = so.split_session(s.xyzi, s.offsets, full.poses, inv, small_maps[0], CRITERIA[criterion], 3, 0.1, pose_offset=2)
    _assert_equal(dev, exp)
