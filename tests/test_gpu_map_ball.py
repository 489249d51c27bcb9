"""The ball subset of the map on the device (ltr_remove_pass_ball): every pass variant, fast-path setting and threshold gives the flags of
the CPU restatement (tests/_ball_oracle.py) bit for bit, on the golden pair, on points one ulp either side of the sphere, and on a
configs[2]-shaped session against per-keyframe subset clouds; the orchestrator and the driver run it in removeOnce / revertOnce only."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import oracle
import lt_mapper_b200 as ltr
from lt_mapper_b200 import removert
import _ball_oracle as B
from test_gpu_scanside_orchestrator import BIN, _PARAMS, _dataset, _n_gpus, _tree

pytestmark = pytest.mark.gpu
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAST = {0: dict(fast_path=False), 1: dict(fast_path=True, cull=False), 2: dict(fast_path=True, cull=True)}
# (device mode, oracle mode, alpha): HD remove, revert at 0.95 r, ND and PD filter passes
VARIANTS = {"HD": (ltr.MODE_HD, oracle.MODE_HD, 2.5), "revert": (ltr.MODE_HD, oracle.MODE_HD, F32(0.95 * F32(2.5))),
            "ND": (ltr.MODE_ND, oracle.MODE_ND, 2.5), "PD": (ltr.MODE_PD, oracle.MODE_PD, 2.5)}
THRESHOLDS = ((0.1, 0.0), (0.1, 0.05))   # (diff_thres, adaptive_coeff): the constant 0.1 m and the adaptive fl(0.05 s)


def _map_for(small_maps, mode):
    return small_maps[0] if mode == ltr.MODE_HD else small_maps[1][::7]   # the filter passes project the other session's map


def _radii(m, poses):
    """two radii (distance quantiles) at which every keyframe's ball holds between 10 and 90 % of the map"""
    d = np.stack([np.sqrt(B.sq_dist(m, c).astype(np.float64)) for c in B.centres(poses)])
    lo, hi = np.quantile(d, 0.1, axis=1).max(), np.quantile(d, 0.9, axis=1).min()
    assert lo < hi, (lo, hi)
    return [float(F32(lo + f * (hi - lo))) for f in (0.25, 0.75)]


def _ball(ctx, m, d, inv, mode, alpha, radius, thres=0.1, coeff=0.0):
    mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(d.xyzi, d.offsets); ps = ctx.poses_upload(d.poses, inv)
    n = ctx.remove_pass_ball(mh, ss, ps, mode, alpha, radius, thres, coeff)
    return ctx.flags_download(mh), n, ctx.last_pass_stats()


# ------------------------------------------------------------------------------------------------------------ 1. golden pair
@pytest.mark.parametrize("fast", [0, 1, 2])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_golden_pair_every_variant(small_pair, small_maps, variant, fast):
    c = small_pair[0]
    mode, omode, alpha = VARIANTS[variant]
    m = _map_for(small_maps, mode)
    inv = oracle.inverse_poses(c.poses)
    with ltr.Context(keyframe_batch=32, **FAST[fast]) as ctx:
        for radius in _radii(m, c.poses):
            for thres, coeff in THRESHOLDS:
                exp = B.remove_pass(m, c.xyzi, c.offsets, c.poses, inv, omode, alpha, radius, thres, coeff)
                got, n, st = _ball(ctx, m, c, inv, mode, alpha, radius, thres, coeff)
                assert n == int(exp.sum()) and np.array_equal(got, exp), (variant, radius, coeff, np.flatnonzero(got != exp)[:8])
                assert exp.sum() > 0
                assert st[0] == len(m) * c.K
                if fast:
                    assert st[1] > 0 and st[1] + st[2] == st[0]


# ------------------------------------------------------------------------------------------------------------ 2. boundary scene
def _shell(rng, c, r2, n):
    """points whose d2 from c is r2 (outside), one ulp below (inside) or one ulp above: ulp walks of points on the sphere"""
    out = []
    R = np.sqrt(np.float64(r2))
    want = {F32(r2), np.nextafter(F32(r2), F32(0)), np.nextafter(F32(r2), F32(np.inf))}
    while len(out) < n:
        v = rng.normal(size=3)
        v[2] *= 0.1   # near the horizon, where the scans see far
        p = (c.astype(np.float64) + R * v / np.linalg.norm(v)).astype(F32)
        for _ in range(64):
            d2 = B.sq_dist(p[None], c)[0]
            if d2 in want:
                out.append(p.copy())
                break
            j = rng.integers(3)
            p[j] = np.nextafter(p[j], F32(np.inf) if (d2 < r2) == (p[j] < c[j]) else F32(-np.inf))
    return np.array(out, F32)


@pytest.mark.parametrize("fast", [0, 1, 2])
def test_boundary_scene(small_pair, small_maps, fast):
    """the golden map plus, for each of the first four keyframes, points on its sphere to the ulp (several keyframes per launch; tiles of
    the map straddle, sit inside and sit outside each ball)"""
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)
    rng = np.random.default_rng(11)
    radius = F32(9.0)
    r2 = B.radius2(radius)
    shells = [_shell(rng, cc, r2, 300) for cc in B.centres(c.poses)[:4]]
    pts = np.concatenate(shells)
    m = np.concatenate([small_maps[0], np.concatenate([pts, np.zeros((len(pts), 1), F32)], 1)])
    cs = B.centres(c.poses)
    for k, s in enumerate(shells):
        d2 = B.sq_dist(s, cs[k])
        assert (d2 == r2).sum() > 20 and (d2 < r2).sum() > 20, k
    with ltr.Context(keyframe_batch=32, **FAST[fast]) as ctx:
        for thres, coeff in THRESHOLDS:
            exp = B.remove_pass(m, c.xyzi, c.offsets, c.poses, inv, oracle.MODE_HD, 2.5, radius, thres, coeff)
            got, n, st = _ball(ctx, m, c, inv, ltr.MODE_HD, 2.5, radius, thres, coeff)
            assert n == int(exp.sum()) and np.array_equal(got, exp), (coeff, np.flatnonzero(got != exp)[:8])
            assert exp[len(small_maps[0]):].sum() > 0, "no shell point flagged: the scene does not test the sphere"
            if fast:
                assert st[6] > 0   # whole tiles outside a ball
        # a NaN point is in no ball and changes nothing
        mn = m.copy()
        mn[5, 0] = np.nan
        exp = B.remove_pass(mn, c.xyzi, c.offsets, c.poses, inv, oracle.MODE_HD, 2.5, radius)
        got, n, _ = _ball(ctx, mn, c, inv, ltr.MODE_HD, 2.5, radius)
        assert np.array_equal(got, exp) and got[5] == 0


# ------------------------------------------------------------------------------------------------------------ 3. huge radius
@pytest.mark.parametrize("fast", [0, 2])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_huge_radius_is_the_full_pass(small_pair, small_maps, variant, fast):
    c = small_pair[0]
    mode, _, alpha = VARIANTS[variant]
    m = _map_for(small_maps, mode)
    inv = oracle.inverse_poses(c.poses)
    with ltr.Context(keyframe_batch=32, **FAST[fast]) as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        n_full = ctx.remove_pass(mh, ss, ps, mode, alpha)
        full = ctx.flags_download(mh)
        n = ctx.remove_pass_ball(mh, ss, ps, mode, alpha, 1e6)
        assert n == n_full and np.array_equal(ctx.flags_download(mh), full)


# ------------------------------------------------------------------------------------------------------------ 4. configs[2] scale
def test_config2_session_against_subset_clouds():
    """100 keyframes of a configs[2]-shaped session (synth), R = 80, fast path 2 with kept images: the ball pass equals the OR of
    ltr_remove_pass over [k, k + 1) on each keyframe's uploaded subset cloud"""
    sys.path.insert(0, ROOT)
    import bench
    blocks = bench.gen_block(0, 100)
    d, inv = blocks[0]
    R = removert.Removerter(num_knn=bench.NUM_KNN, knn_thr=bench.KNN_THR)
    for s, (ds, invs) in enumerate(blocks):
        R.load_session(s, ds.xyzi, ds.offsets, ds.poses, invs)
    R.run_step0()
    m = R.ctx.cloud_download(R.cloud_handle("map_global_curr_", 0))
    R.close()
    radius = 80.0
    cs = B.centres(d.poses)
    with ltr.Context(keyframe_batch=32, fast_path=True, cull=True) as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(d.xyzi, d.offsets); ps = ctx.poses_upload(d.poses, inv)
        n = ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, radius)
        got = ctx.flags_download(mh)
        st = ctx.last_pass_stats()
        exp = np.zeros(len(m), np.uint8)
        for k in range(d.K):
            idx = np.flatnonzero(B.members(m, cs[k], radius))
            sh = ctx.cloud_upload(m[idx])
            ctx.remove_pass(sh, ss, ps, ltr.MODE_HD, 2.5, kf_begin=k, kf_end=k + 1)
            exp[idx[ctx.flags_download(sh) != 0]] = 1
            ctx.cloud_free(sh)
    assert len(m) > 500_000 and exp.sum() > 0
    assert n == int(exp.sum()) and np.array_equal(got, exp), np.flatnonzero(got != exp)[:8]
    assert st[6] > 0.3 * st[0], st   # most pairs are outside the balls


# ------------------------------------------------------------------------------------------------------------ 5. kept images
@pytest.mark.parametrize("cache_mb", ["0", None])
def test_kept_images_ball_full_ball(small_pair, small_maps, monkeypatch, cache_mb):
    if cache_mb is None:
        monkeypatch.delenv("LTR_SCAN_IMAGE_CACHE_MB", raising=False)
    else:
        monkeypatch.setenv("LTR_SCAN_IMAGE_CACHE_MB", cache_mb)
    c = small_pair[0]
    m = small_maps[0]
    inv = oracle.inverse_poses(c.poses)
    radius = _radii(m, c.poses)[0]
    calls = [(radius, 0.0), (None, 0.0), (radius, 0.0), (radius, 0.05), (None, 0.05), (radius, 0.0)]

    def one(ctx, mh, ss, ps, r, coeff):
        if r is None:
            if coeff:
                ctx.remove_pass_adaptive(mh, ss, ps, ltr.MODE_HD, 2.5, coeff)
            else:
                ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)
        else:
            ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, r, 0.1, coeff)
        return ctx.flags_download(mh)

    fresh = {}
    for call in set(calls):
        with ltr.Context() as ctx:
            fresh[call] = one(ctx, ctx.cloud_upload(m), ctx.scanset_upload(c.xyzi, c.offsets), ctx.poses_upload(c.poses, inv), *call)
    assert not np.array_equal(fresh[(None, 0.0)], fresh[(radius, 0.0)])
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        for call in calls:   # warm-up: the flag array, the kept sets and the allocator's blocks
            one(ctx, mh, ss, ps, *call)
        for call in calls:
            base = ctx.memory_stats()[0]
            assert np.array_equal(one(ctx, mh, ss, ps, *call), fresh[call]), call
            assert ctx.memory_stats()[0] == base, call


# ------------------------------------------------------------------------------------------------------------ 6. bad input
def test_bad_radii_and_coefficients(small_pair, small_maps):
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(small_maps[0]); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)   # the flag array of the map is allocated by its first pass
        ctx.scan_images_release(True)
        base = ctx.memory_stats()[0]
        bad = [(r, 0.0) for r in (0.0, -0.0, -1.0, float("nan"), float("inf"), float("-inf"))]
        bad += [(80.0, k) for k in (-0.05, 1.0, 2.0, float("nan"), float("inf"))]
        for r, coeff in bad:
            with pytest.raises(ltr.LtrError) as e:
                ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, r, 0.1, coeff)
            assert e.value.code == -1, (r, coeff)
        assert ctx.memory_stats()[0] == base
        for mode in (ltr.MODE_HD, ltr.MODE_ND, ltr.MODE_PD):
            ctx.remove_pass_ball(mh, ss, ps, mode, 2.5, 20.0)
            ctx.remove_pass_ball(mh, ss, ps, mode, 2.5, 20.0, 0.1, 0.05)
        ctx.scan_images_release(True)
        assert ctx.memory_stats()[0] == base
        # a radius whose square rounds to 0 admits no point
        assert ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, 1e-30) == 0


# ------------------------------------------------------------------------------------------------------------ 7. orchestrator
def _step1(small_pair, radius, schedule=((removert.OP_REMOVE, 2.5),)):
    c, q = small_pair
    G = removert.Removerter(num_knn=2, knn_thr=0.01, schedule=schedule)
    if radius is not None:
        G.set_map_ball(radius)
    G.load_session(0, c.xyzi, c.offsets, c.poses, oracle.inverse_poses(c.poses))
    G.load_session(1, q.xyzi, q.offsets, q.poses, oracle.inverse_poses(q.poses))
    G.run_step0()
    G.stage("makeGlobalMap")
    M = G.cloud("map_global_curr_", 0)
    G.stage("removeHighDynamicPoints")
    out = (M, G.log(), G.cloud("map_global_curr_static_", 0), G.cloud("map_global_curr_dynamic_", 0))
    G.close()
    return out


def test_orchestrator_runs_the_ball_in_removeOnce(small_pair, small_maps):
    """Step 1's removeOnce(2.5) with set_map_ball(R): the pass log and the static map equal a replay through Context.remove_pass_ball,
    apply_partition and the voxeliser on the orchestrator's own map; set_map_ball(0) gives the default outputs byte for byte."""
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)
    radius = _radii(small_maps[0], c.poses)[0]
    M, log, static, dynamic = _step1(small_pair, radius)
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(M); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        n = ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, radius)
        sh, dh = ctx.apply_partition(mh)
        exp_static = ctx.cloud_download(ctx.voxel_centroid(sh, 0.05))
    assert log[0][0] == "removeOnce" and log[0][1] == len(M) and log[0][2] == n, log[0]
    assert n == int(B.remove_pass(M, c.xyzi, c.offsets, c.poses, inv, oracle.MODE_HD, 2.5, radius).sum())
    assert static.shape == exp_static.shape and np.array_equal(static.view(np.uint32), exp_static.view(np.uint32))
    default = _step1(small_pair, None)
    off = _step1(small_pair, 0.0)
    assert log[0][2] != default[1][0][2]
    for a, b in zip(default, off):
        if isinstance(a, np.ndarray):
            assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
        else:
            assert a == b


_TRACE_SCRIPT = """
import sys, numpy as np
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import oracle, synth
from lt_mapper_b200 import removert
c, q = synth.make_pair(6, beams=32, az_steps=900)
G = removert.Removerter(num_knn=2, knn_thr=0.01, schedule={schedule!r})
G.set_map_ball(20.0)
G.load_session(0, c.xyzi, c.offsets, c.poses, oracle.inverse_poses(c.poses))
G.load_session(1, q.xyzi, q.offsets, q.poses, oracle.inverse_poses(q.poses))
G.run_step0(); G.run_step12(); G.run_step3()
print("LOG", [e[0] for e in G.log()])
G.close()
"""


def test_orchestrator_trace_counts():
    """under LTR_TRACE=1 the context's entry-point totals show one ltr_remove_pass_ball per selfRemovert pass of both sessions, and the
    six ND / PD filter passes still on ltr_remove_pass"""
    schedule = ((removert.OP_REMOVE, 2.5), (removert.OP_REVERT, float(F32(0.95 * F32(2.5)))), (removert.OP_REMOVE, 2.5))
    script = _TRACE_SCRIPT.format(root=ROOT, tests=os.path.dirname(os.path.abspath(__file__)), schedule=schedule)
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=600, env=dict(os.environ, LTR_TRACE="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    calls = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[ltr trace\] (\S+)\s+calls\s+(\d+)", r.stderr)}
    log = eval(re.search(r"LOG (\[.*\])", r.stdout).group(1))
    hd = sum(1 for e in log if e in ("removeOnce", "revertOnce"))
    assert hd == 2 * len(schedule), log
    assert calls.get("ltr_remove_pass_ball") == hd, calls
    assert calls.get("ltr_remove_pass") == 6, calls
    assert sum(1 for e in log if e in ("iremoveOnceForND", "removeOnceForPD")) == 6, log


def test_orchestrator_rejects_bad_radii():
    with removert.Removerter() as G:
        for bad in (-1.0, float("nan"), float("inf"), float("-inf")):
            with pytest.raises(Exception):
                G.set_map_ball(bad)
        G.set_map_ball(80.0)
        G.set_map_ball(0.0)


# ------------------------------------------------------------------------------------------------------------ 8. driver
SUMMARY = re.compile(r" Map ball: radius ([0-9.e+-]+) m")


def _drive(tmp_path, tag, args, world=1):
    out = tmp_path / f"out_{tag}"
    cfg = tmp_path / f"params_{tag}.yaml"
    cfg.write_text(_PARAMS.format(out=out, d=tmp_path))
    logs, procs = [], []
    for rank in range(world):
        e = dict(os.environ, RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), LTR_NCCL_ID_FILE=str(tmp_path / f"nccl_{tag}"))
        procs.append(subprocess.Popen([BIN, "--config", str(cfg)] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=e))
    for p in procs:
        o, _ = p.communicate(timeout=600)
        assert p.returncode == 0, o
        logs.append(o)
    return out, "".join(logs)


@pytest.mark.parametrize("flag,radius", [("--map-ball", 80.0), ("--map-ball=15", 15.0)])
def test_driver_writes_what_the_orchestrator_holds(tmp_path, small_pair, flag, radius):
    _dataset(tmp_path, small_pair)
    out_plain, log_plain = _drive(tmp_path, "plain", [])
    out, log = _drive(tmp_path, "ball", [flag])
    plain, ball = _tree(out_plain), _tree(out)
    assert set(plain) == set(ball), "the option must not change the output tree's layout"
    assert not SUMMARY.search(log_plain) and float(SUMMARY.search(log).group(1)) == pytest.approx(radius)
    c, q = small_pair
    kc = removert.parse_keyframes(c.K, 2, 5, 1)
    kq = removert.parse_keyframes_in_roi(q.poses, c.poses[kc], 1)
    G = removert.Removerter(num_knn=3, knn_thr=0.1)
    G.set_map_ball(radius)
    for s, d, ks in ((0, c, kc), (1, q, kq)):
        xyzi = np.concatenate([d.scan(k) for k in ks])
        off = np.concatenate([[0], np.cumsum([len(d.scan(k)) for k in ks])])
        poses = removert.read_poses(str(tmp_path / ("central" if s == 0 else "query") / "poses.txt"))[ks]
        G.load_session_raw(s, xyzi, off, poses, removert.inverse_poses(poses))
    G.run_step0()
    G.run_step12()
    G.run_step3()
    compared = []
    for rel in ball:
        if "/" in rel or not rel.endswith(".pcd"):
            continue
        try:
            exp = G.cloud("saved:" + rel[:-4])
        except Exception:  # noqa: BLE001 -- files that are not saved maps of the orchestrator
            continue
        got = removert.read_pcd(str(out / rel))
        assert got.shape == exp.shape and np.array_equal(got.view(np.uint32), exp.view(np.uint32)), rel
        compared.append(rel)
    assert {"nd_map.pcd", "pd_map.pcd"} <= set(compared), compared
    if radius < 80.0:
        assert any(ball[k] != plain[k] for k in compared), "the ball changed nothing"
    G.close()


@pytest.mark.parametrize("value", ["0", "-1", "nan", "inf", "-inf", "abc", "80x", ""])
def test_driver_bad_value_exits_2(tmp_path, value):
    r = subprocess.run([BIN, "--config", str(tmp_path / "unused.yaml"), "--map-ball=" + value], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2, r.stdout + r.stderr


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
def test_driver_two_ranks(tmp_path, small_pair):
    _dataset(tmp_path, small_pair)
    out1, _ = _drive(tmp_path, "one", ["--map-ball=15"])
    out2, _ = _drive(tmp_path, "two", ["--map-ball=15"], world=2)
    one, two = _tree(out1), _tree(out2)
    assert set(one) == set(two)
    for k in one:
        assert one[k] == two[k], k
