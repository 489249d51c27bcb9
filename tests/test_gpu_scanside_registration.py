"""Scan-side removal between sessions with ICP fine registration on the GPU (ltr_icp_refine_scanside, ltr_scanside_split_refined; icp.cu,
scanside.cu), through the host orchestrator (ltrh_scanside_removal_registered, ltrh_scanside_icp_stats) and the drop-in driver
(--clean-scans-between), against the CPU restatement (tests/_scanside_reg_oracle.py) bit for bit."""
import os
import re

import numpy as np
import pytest

import oracle
import _scanside_oracle as so
import _scanside_reg_oracle as sro
from lt_mapper_b200 import removert
from test_gpu_icp import _perturb
from test_gpu_scanside_orchestrator import BIN, _dataset, _n_gpus, _tree
from test_gpu_icp_driver import _run as _driver

pytestmark = pytest.mark.gpu
CRITERIA = [so.MAP, so.SCAN_MINUS_MAP]
SUMMARY = re.compile(r" Scan-side registration: (\d+) of (\d+) keyframes accepted, median iterations (\d+)")
L2B = np.array([[np.cos(0.05), 0, np.sin(0.05), 0.3], [0, 1, 0, -0.02], [-np.sin(0.05), 0, np.cos(0.05), 1.1], [0, 0, 0, 1]])


def _per_kf(pts, off):
    return [pts[off[j]:off[j + 1]] for j in range(len(off) - 1)]


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _icp_equal(got, exp):
    T, fit, it, ex = got
    eT, efit, eit, eex = exp
    assert np.array_equal(it, eit) and np.array_equal(ex, eex), (it, eit, ex, eex)
    assert _same(T, eT), np.abs(T - eT).max()
    assert _same(fit, efit), (fit, efit)


def _download_parts(ctx, pair):
    out = []
    for h in pair:
        out.append(_per_kf(*ctx.scanset_download(h)))
        ctx.scanset_free(h)
    return out


def _parts_equal(got, exp, what=""):
    for part in range(2):
        assert len(got[part]) == len(exp[part])
        for kf, (a, b) in enumerate(zip(got[part], exp[part])):
            assert _same(a, b), (what, part, kf, a.shape, b.shape)


@pytest.mark.parametrize("perturbed", [False, True])
@pytest.mark.parametrize("pair", ["CQ", "QC"])
def test_icp_refine_scanside_matches_the_oracle(small_pair, small_maps, pair, perturbed):
    """(map, scan) = (C,Q) and (Q,C), with the synthetic poses and with a 0.3 m / 1 degree error; with the identity extrinsic the entry
    equals ltr_icp_refine byte for byte."""
    import lt_mapper_b200 as ltr
    s = small_pair["CQ".index(pair[1])].subset(0, 3)
    poses = _perturb(s.poses) if perturbed else s.poses
    md = oracle.voxel(small_maps["CQ".index(pair[0])], 0.4)
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        ss = ctx.scanset_upload(s.xyzi, s.offsets)
        ps = ctx.poses_upload(poses, oracle.inverse_poses(poses))
        td = ctx.cloud_upload(md)
        got = ctx.icp_refine_scanside(ss, ps, td)
        _icp_equal(got, sro.register_session(s.xyzi, s.offsets, poses, md))
        _icp_equal(got, ctx.icp_refine(ss, ps, td))
        if perturbed:
            assert (got[1] < 1.0).any()
        ctx.scanset_free(ss)
        ctx.poses_free(ps)
        ctx.cloud_free(td)
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0


@pytest.mark.parametrize("order", [0, 1])
def test_icp_refine_scanside_with_an_extrinsic(small_pair, small_maps, order):
    """A non-identity LiDAR extrinsic, both transform orders: the scan goes to the global frame with lidar2base, as scan-side removal moves
    it, and the result equals the oracle, not ltr_icp_refine."""
    import lt_mapper_b200 as ltr
    b2l = oracle.inverse4x4(L2B)
    full = small_pair[1]
    s = full.subset(1, 3)
    poses = _perturb(full.poses, 0.2, 0.5)
    md = oracle.voxel(small_maps[0], 0.4)
    with ltr.Context(device=0, lidar2base=L2B, base2lidar=b2l, transform_order=order) as ctx:
        ss = ctx.scanset_upload(s.xyzi, s.offsets)
        ps = ctx.poses_upload(poses, oracle.inverse_poses(poses))
        td = ctx.cloud_upload(md)
        got = ctx.icp_refine_scanside(ss, ps, td, pose_offset=1)
        _icp_equal(got, sro.register_session(s.xyzi, s.offsets, poses, md, L2B, order, pose_offset=1))
        assert not _same(got[0], ctx.icp_refine(ss, ps, td, pose_offset=1)[0])
        ctx.scanset_free(ss)
        ctx.poses_free(ps)
        ctx.cloud_free(td)


def _split_check(ctx, xyzi, offsets, poses, m, crit, T, acc, k=3, thr=0.1, pose_offset=0, l2b=oracle.IDENTITY, order=0):
    """ltr_scanside_split_refined against the oracle; keyframes with acc == 0 also against ltr_scanside_split."""
    b2l = oracle.IDENTITY if l2b is oracle.IDENTITY else oracle.inverse4x4(l2b)
    inv = oracle.inverse_poses(poses)
    ss = ctx.scanset_upload(xyzi, offsets)
    ps = ctx.poses_upload(poses, inv)
    mh = ctx.cloud_upload(m)
    got = _download_parts(ctx, ctx.scanside_split_refined(ss, ps, mh, crit, k, thr, T, acc, pose_offset=pose_offset))
    plain = _download_parts(ctx, ctx.scanside_split(ss, ps, mh, crit, k, thr, pose_offset=pose_offset))
    exp = sro.split_session_refined(xyzi, offsets, poses, inv, m, crit, k, thr, T, acc, l2b, b2l, order, pose_offset)
    _parts_equal(got, exp, "oracle")
    for kf in range(len(offsets) - 1):
        if not acc[kf]:
            assert _same(got[0][kf], plain[0][kf]) and _same(got[1][kf], plain[1][kf]), ("rejected keyframe", kf)
    ctx.scanset_free(ss)
    ctx.poses_free(ps)
    ctx.cloud_free(mh)
    return got, plain


@pytest.mark.parametrize("criterion", CRITERIA)
def test_split_refined_matches_the_oracle(small_pair, small_maps, criterion, monkeypatch):
    """A mixed accept mask on registered query keyframes (0.3 m / 1 degree error) against the central map; every keyframe rejected gives
    ltr_scanside_split; a pose table indexed with pose_offset, empty keyframes, and launches of a few keyframes each."""
    import lt_mapper_b200 as ltr
    full = small_pair[1]
    q = full.subset(0, 3)
    poses = _perturb(full.poses)
    m = small_maps[0]
    md = oracle.voxel(m, 0.4)
    T, fit, _, _ = sro.register_session(q.xyzi, q.offsets, poses, md)
    acc = np.array([True, False, True]) & (fit < 1.0)
    assert acc.any() and not acc.all()
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        got, plain = _split_check(ctx, q.xyzi, q.offsets, poses, m, criterion, T, acc)
        assert sum(len(a) for a in got[0]) > sum(len(a) for a in plain[0]), "registration must keep more static points"
        _split_check(ctx, q.xyzi, q.offsets, poses, m, criterion, T, np.zeros(3, bool))
        # keyframes 2..4 of the full pose table, the first of them empty
        s = full.subset(2, 5)
        xyzi = s.xyzi[s.offsets[1]:]
        offsets = np.concatenate([[0], s.offsets[1:] - s.offsets[1]]).astype(np.int64)
        T2 = np.tile(np.eye(4, dtype=np.float32), (3, 1, 1))
        T2[1] = T[0]
        T2[2] = T[2]
        _split_check(ctx, xyzi, offsets, poses, m, criterion, T2, np.array([1, 1, 0], bool), pose_offset=2)
        for chunk in ("1", "60000"):
            monkeypatch.setenv("LTR_SCANSIDE_CHUNK_POINTS", chunk)
            _split_check(ctx, q.xyzi, q.offsets, poses, m, criterion, T, acc)
        monkeypatch.delenv("LTR_SCANSIDE_CHUNK_POINTS")
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0


def test_split_refined_with_an_extrinsic(small_pair, small_maps):
    import lt_mapper_b200 as ltr
    c = small_pair[0].subset(0, 2)
    T = np.tile(np.eye(4, dtype=np.float32), (2, 1, 1))
    T[0, :3, 3] = [0.05, -0.03, 0.01]
    with ltr.Context(device=0, lidar2base=L2B, base2lidar=oracle.inverse4x4(L2B), transform_order=1) as ctx:
        for crit in CRITERIA:
            _split_check(ctx, c.xyzi, c.offsets, c.poses, small_maps[1], crit, T, np.array([1, 0], bool), l2b=L2B, order=1)


def test_split_refined_rejections():
    import lt_mapper_b200 as ltr
    scan = np.array([[1, 2, 3, 0], [4, 5, 6, 0]], np.float32)
    off = np.array([0, 2], np.int64)
    pose = np.eye(4)[None]
    T = np.eye(4, dtype=np.float32)[None]
    with ltr.Context(device=0) as ctx:
        live0 = ctx.memory_stats()[0]
        ss = ctx.scanset_upload(scan, off)
        ps = ctx.poses_upload(pose, pose)
        good = ctx.cloud_upload(scan)
        bad = ctx.cloud_upload(np.array([[0, 0, 0, 0], [np.nan, 0, 0, 0], [1, 1, 1, 0]], np.float32))
        empty = ctx.cloud_upload(np.zeros((0, 4), np.float32))
        bad_scan = ctx.scanset_upload(np.array([[np.inf, 0, 0, 0]], np.float32), np.array([0, 1], np.int64))
        for crit in CRITERIA:
            for args in ((ss, ps, good, crit, 3, 0.1, None, [1]), (ss, ps, good, crit, 3, 0.1, T, None),    # null tables
                         (ss, ps, good, crit, 0, 0.1, T, [1]), (ss, ps, good, crit, 17, 0.1, T, [1]),       # bad k
                         (ss, ps, good, crit, 3, 0.0, T, [1]), (ss, ps, good, crit, 3, float("nan"), T, [1]),   # bad thr
                         (ss, ps, bad, crit, 3, 0.1, T, [1]), (bad_scan, ps, good, crit, 3, 0.1, T, [1]),   # non-finite input
                         (ss, ps, empty, crit, 3, 0.1, T, [1])):
                with pytest.raises(ltr.LtrError):
                    ctx.scanside_split_refined(*args)
            with pytest.raises(ltr.LtrError):
                ctx.scanside_split_refined(ss, ps, good, crit, 3, 0.1, T, [1], pose_offset=1)
            # a transform that moves the scan to infinity fails the finite check
            with pytest.raises(ltr.LtrError):
                ctx.scanside_split_refined(ss, ps, good, crit, 3, 0.1, np.full((1, 4, 4), np.inf, np.float32), [1])
        with pytest.raises(ltr.LtrError):
            ctx.icp_refine_scanside(ss, ps, empty)
        with pytest.raises(ltr.LtrError):
            ctx.icp_refine_scanside(bad_scan, ps, good)
        for h in (good, bad, empty):
            ctx.cloud_free(h)
        for h in (ss, bad_scan):
            ctx.scanset_free(h)
        ctx.poses_free(ps)
        ctx.synchronize()
        assert ctx.memory_stats()[0] == live0


def test_orchestrator_matches_the_oracle_and_keeps_step2_stats(small_pair):
    """ltrh_scanside_removal_registered for (C,Q) and (Q,C) on a query session with a pose error equals the restatement on the
    orchestrator's own inputs; its registration comes back through ltrh_scanside_icp_stats, and the ICP-refined Step 2's ltrh_icp_stats
    is unchanged by it.  A plain scan-side removal, a failed registered one and ltrh_reset_to_step0 empty the registration stats."""
    c, q = (s.subset(0, 3) for s in small_pair)
    qp = _perturb(q.poses)
    G = removert.Removerter(num_knn=3, knn_thr=0.1)
    G.set_icp_refinement(True)
    G.load_session(0, c.xyzi, c.offsets, c.poses, oracle.inverse_poses(c.poses))
    G.load_session(1, q.xyzi, q.offsets, qp, oracle.inverse_poses(qp))
    G.run_step0()
    G.run_step12()
    step2 = [G.icp_stats(s) for s in (0, 1)]
    assert step2[0]["fitness"].size == 3
    for crit, (m_sess, s_sess) in ((so.SCAN_MINUS_MAP, (0, 1)), (so.MAP, (1, 0))):
        poses = (c.poses, qp)[s_sess]
        G.scanside_removal_registered(m_sess, s_sess, crit)
        scans, off = G.scanset("keyframe_scans_", s_sess)
        m = G.cloud("map_global_curr_static_", m_sess)
        (est, edy), (T, fit, it, ex, acc) = sro.removal_registered(scans, off, poses, oracle.inverse_poses(poses), m, crit, 3, 0.1)
        st = G.scanside_icp_stats(s_sess)
        _icp_equal((st["T"], st["fitness"], st["iterations"], st["exit"]), (T, fit, it, ex))
        assert np.array_equal(st["accepted"], acc)
        for member, exp in (("scans_static_", est), ("scans_dynamic_", edy)):
            got = _per_kf(*G.scanset(member, s_sess))
            assert len(got) == len(exp)
            for kf, (a, b) in enumerate(zip(got, exp)):
                assert _same(a, b), (crit, m_sess, s_sess, member, kf)
    assert G.scanside_icp_stats(1)["accepted"].any()
    for s in (0, 1):
        after = G.icp_stats(s)
        for key in step2[s]:
            assert _same(after[key], step2[s][key]), (s, key)
    G.scanside_removal(0, 1, so.MAP)
    assert G.scanside_icp_stats(1)["fitness"].size == 0 and G.scanside_icp_stats(0)["fitness"].size == 3
    # a removal whose registration succeeds but whose split fails (unknown criterion) leaves no registration stats behind
    with pytest.raises(Exception):
        G.scanside_removal_registered(1, 0, 7)
    assert G.scanside_icp_stats(0)["fitness"].size == 0
    G.reset_to_step0()
    assert G.scanside_icp_stats(0)["fitness"].size == 0
    G.close()


@pytest.mark.parametrize("flag,crit", [("--clean-scans-between", so.MAP), ("--clean-scans-between=scan-minus-map", so.SCAN_MINUS_MAP)])
def test_driver_clean_scans_between(tmp_path, small_pair, flag, crit):
    """The four new directories hold, under the input scans' names, what the orchestrator's registered removal (checked against the
    restatement above) holds for the driver's keyframe selection; every other file equals a run without the flag; the summary line reports
    the orchestrator's registrations; --clean-scans combines with it; --compose rejects it."""
    import subprocess
    _dataset(tmp_path, small_pair)
    out_plain, log_plain = _driver(tmp_path, "plain", [])
    out, log = _driver(tmp_path, "between", [flag, "--clean-scans"])
    plain, between = _tree(out_plain), _tree(out)
    assert not SUMMARY.search(log_plain)
    m = SUMMARY.search(log)
    assert m, log
    dirs = ("scan_static/query_vs_central/", "scan_dynamic/query_vs_central/", "scan_static/central_vs_query/", "scan_dynamic/central_vs_query/")
    others = {k: v for k, v in between.items() if not k.startswith(dirs)}
    assert {k: v for k, v in others.items() if k in plain} == plain
    assert all(k.startswith(("scan_static/central/", "scan_static/query/", "scan_dynamic/central/", "scan_dynamic/query/", "map_static/",
                             "map_dynamic/")) for k in set(others) - set(plain))
    c, q = small_pair
    kc = removert.parse_keyframes(c.K, 2, 5, 1)
    kq = removert.parse_keyframes_in_roi(q.poses, c.poses[kc], 1)
    G = removert.Removerter(num_knn=3, knn_thr=0.1)
    for s, d, ks in ((0, c, kc), (1, q, kq)):
        xyzi = np.concatenate([d.scan(k) for k in ks])
        off = np.concatenate([[0], np.cumsum([len(d.scan(k)) for k in ks])])
        poses = removert.read_poses(str(tmp_path / ("central" if s == 0 else "query") / "poses.txt"))[ks]
        G.load_session_raw(s, xyzi, off, poses, removert.inverse_poses(poses))
    G.run_step0()
    G.run_step12()
    G.run_step3()
    its, accepted = [], 0
    for s_sess, name, ks in ((1, "query_vs_central", kq), (0, "central_vs_query", kc)):
        G.scanside_removal_registered(1 - s_sess, s_sess, crit)
        st = G.scanside_icp_stats(s_sess)
        its += list(st["iterations"])
        accepted += int(st["accepted"].sum())
        for member, sub in (("scans_static_", "scan_static"), ("scans_dynamic_", "scan_dynamic")):
            exp = _per_kf(*G.scanset(member, s_sess))
            files = sorted(os.listdir(out / sub / name))
            assert files == [f"{k:06d}.pcd" for k in ks]
            for fn, e in zip(files, exp):
                got = removert.read_pcd(str(out / sub / name / fn))
                assert _same(got, e), (sub, name, fn)
    its = np.sort(its)
    assert (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (accepted, len(its), int(its[(len(its) - 1) // 2]))
    G.close()
    cfg = tmp_path / "params_plain.yaml"
    r = subprocess.run([BIN, "--config", str(cfg), flag, f"--compose={out_plain}"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 2 and "--clean-scans-between" in r.stderr, r.stderr


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("split", [True, False])
def test_driver_clean_scans_between_two_ranks(tmp_path, small_pair, split):
    """Each rank registers and splits its own keyframe block against its replica of the other map, with no collective: the tree and the
    summary line equal the single-process run."""
    _dataset(tmp_path, small_pair)
    args = ["--clean-scans-between=scan-minus-map"] + ([] if split else ["--no-split"])
    out1, log1 = _driver(tmp_path, "one", args)
    out2, log2 = _driver(tmp_path, "two", args, world=2)
    assert SUMMARY.search(log1).groups() == SUMMARY.search(log2).groups()
    one, two = _tree(out1), _tree(out2)
    assert set(one) == set(two)
    for k in one:
        assert one[k] == two[k], k
