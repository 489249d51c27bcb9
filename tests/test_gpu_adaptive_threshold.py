"""The range-adaptive discrepancy threshold on the device (ltr_remove_pass_adaptive): every pass variant, every fast-path setting and
the kept scan images give the flags of the CPU restatement (tests/_adaptive_oracle.py) bit for bit, on the small golden pair, on a scene
built on the edge of the rule, at the azimuth seam, and at the tile-cull bound; the orchestrator and the driver apply it to every pass."""
import os
import re
import subprocess

import numpy as np
import pytest

import oracle
import lt_mapper_b200 as ltr
from lt_mapper_b200 import removert
import _adaptive_oracle as A
from test_gpu_project_seam import _scan_set, seam_scene
from test_gpu_scanside_orchestrator import BIN, _PARAMS, _dataset, _n_gpus, _tree

pytestmark = pytest.mark.gpu
F32 = np.float32
COEFFS = (0.01, 0.05, 0.2)
FAST = {0: dict(fast_path=False), 1: dict(fast_path=True, cull=False), 2: dict(fast_path=True, cull=True)}
# (device mode, oracle mode, alpha): HD remove, revert at 0.95 r, ND and PD filter passes
VARIANTS = {"HD": (ltr.MODE_HD, oracle.MODE_HD, 2.5), "revert": (ltr.MODE_HD, oracle.MODE_HD, F32(0.95 * F32(2.5))),
            "ND": (ltr.MODE_ND, oracle.MODE_ND, 2.5), "PD": (ltr.MODE_PD, oracle.MODE_PD, 2.5)}


def _run(ctx, m, xyzi, off, poses, inv, mode, alpha, coeff):
    mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(xyzi, off); ps = ctx.poses_upload(poses, inv)
    n = ctx.remove_pass_adaptive(mh, ss, ps, mode, alpha, coeff)
    return ctx.flags_download(mh), n, ctx.last_pass_stats()


# ------------------------------------------------------------------------------------------------------------ 1. golden pair
@pytest.mark.parametrize("fast", [0, 1, 2])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_golden_pair_every_variant(small_pair, small_maps, variant, fast):
    c = small_pair[0]
    mode, omode, alpha = VARIANTS[variant]
    m = small_maps[0] if mode == ltr.MODE_HD else small_maps[1][::7]   # the filter passes project the other session's map
    inv = oracle.inverse_poses(c.poses)
    with ltr.Context(keyframe_batch=32, **FAST[fast]) as ctx:
        for coeff in COEFFS:
            exp = A.remove_pass(m, c.xyzi, c.offsets, inv, omode, alpha, coeff)
            got, n, _ = _run(ctx, m, c.xyzi, c.offsets, c.poses, inv, mode, alpha, coeff)
            assert n == int(exp.sum()) and np.array_equal(got, exp), (variant, coeff, np.flatnonzero(got != exp)[:8])
            assert exp.sum() > 0
        # the constant threshold is untouched by the adaptive passes around it
        const = oracle.remove_pass(m, c.xyzi, c.offsets, inv, omode, alpha)
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        assert ctx.remove_pass(mh, ss, ps, mode, alpha) == int(const.sum()) and np.array_equal(ctx.flags_download(mh), const)


# ------------------------------------------------------------------------------------------------------------ 2. threshold edge
def _pixel_centre_dirs(rng, n, alpha, vfov=50.0, hfov=360.0):
    rows, cols = ltr.reset_rimg_size(alpha, vfov, hfov)
    px = rng.choice(rows * cols, n, replace=False)
    r, c = px // cols, px % cols
    az = np.deg2rad(c * hfov / cols - 0.5 * hfov)
    el = np.deg2rad((1.0 - r / rows) * vfov - 0.5 * vfov)
    keep = (np.abs(az) < np.deg2rad(179.0)) & (np.abs(el) < np.deg2rad(0.5 * vfov - 1.0))
    az, el = az[keep], el[keep]
    return np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1)


def _range(p):
    p = p.astype(F32)
    return np.sqrt((p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1]) + p[..., 2] * p[..., 2])   # cart2sph's r in f32 (utility.cpp:48)


def _edge_point(d, s, coeff, nd, side):
    """A map point on direction d whose range rho has fl(s - rho) (nd: fl(rho - s)) just above t = fl(coeff s) (side 0) or at / just
    below it (side 1): consecutive float scalings of d, so the two sides are one or two ulps of rho apart."""
    t = F32(F32(coeff) * s)
    target = F32(s + t) if nd else F32(s - t)
    lam = np.nextafter(target, F32(-np.inf))
    for _ in range(6):
        lam = np.nextafter(lam, F32(-np.inf))
    pts, diffs = [], []
    for _ in range(14):
        p = (d * np.float64(lam)).astype(F32)
        rho = _range(p)
        pts.append(p); diffs.append(F32(rho - s) if nd else F32(s - rho))
        lam = np.nextafter(lam, F32(np.inf))
    above = [i for i, v in enumerate(diffs) if v > t]
    below = [i for i, v in enumerate(diffs) if v <= t]
    assert above and below
    return pts[(min(above) if nd else max(above))] if side == 0 else pts[(max(below) if nd else min(below))]


def edge_scene(seed, coeff, K=4, n=3000, alpha=1.0):
    """K identity keyframes, one map point per ray at a pixel centre, each ray owned by one keyframe (the only one with a scan return
    there): the map point sits one ulp inside or outside the edge of the rule, in front of the return (HD / PD) or behind it (ND)."""
    rng = np.random.default_rng(seed)
    dirs = _pixel_centre_dirs(rng, n, alpha)
    s = rng.uniform(1.0, 150.0, len(dirs)).astype(F32)
    scan_pts = (dirs * s[:, None]).astype(F32)
    s = _range(scan_pts)                                              # the scan image's value at the pixel
    owner = np.arange(len(dirs)) % K
    nd = rng.random(len(dirs)) < 0.5
    side = rng.integers(0, 2, len(dirs))
    m = np.stack([_edge_point(dirs[i], s[i], coeff, nd[i], side[i]) for i in range(len(dirs))])
    scans = [np.concatenate([scan_pts[owner == k], np.zeros((int((owner == k).sum()), 1), F32)], 1) for k in range(K)]
    xyzi, off = _scan_set(scans)
    poses = np.repeat(np.eye(4)[None], K, 0)
    return np.concatenate([m, np.ones((len(m), 1), F32)], 1), xyzi, off, poses, nd, side


@pytest.mark.parametrize("coeff", [0.05, 0.0625, 0.2])
def test_threshold_edge_scene(coeff):
    m, xyzi, off, poses, nd, side = edge_scene(11, coeff)
    inv = poses.copy()
    for mode, omode in ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_PD, oracle.MODE_PD), (ltr.MODE_ND, oracle.MODE_ND)):
        exp = A.remove_pass(m, xyzi, off, inv, omode, 1.0, coeff)
        want = (~nd & (side == 0)) if omode != oracle.MODE_ND else (nd & (side == 0))
        assert np.array_equal(exp.astype(bool), want), "the scene is not on the edge it was built for"
        for fast in FAST:
            with ltr.Context(keyframe_batch=32, **FAST[fast]) as ctx:
                got, n, st = _run(ctx, m, xyzi, off, poses, inv, mode, 1.0, coeff)
            assert np.array_equal(got, exp), (mode, fast, np.flatnonzero(got != exp)[:8])
            if fast and omode != oracle.MODE_ND:
                assert st[2] >= (~nd).sum(), "pairs on the edge must reach the exact path"


# ------------------------------------------------------------------------------------------------------------ 3. azimuth seam
@pytest.mark.parametrize("hfov", [360.0, 359.0])
def test_seam_scene(hfov):
    """The guard-padded variant (360 degrees) and the unpadded short-elevation variant (359 degrees), batches of 32 and 3."""
    m, scans, poses, inv, owner = seam_scene(4, 8, 50.0, nonrigid=(5,), nonfinite=True)
    xyzi, off = _scan_set(scans)
    fin = np.isfinite(m[:, :3]).all(1)
    bad = []
    for mode, omode in ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_PD, oracle.MODE_PD), (ltr.MODE_ND, oracle.MODE_ND)):
        for alpha in (2.5, 1.0):
            exp = np.zeros(len(m), np.uint8)
            exp[fin] = A.remove_pass(m[fin], xyzi, off, inv, omode, alpha, 0.05, hfov=hfov)
            assert exp.sum() > 0
            for B in (32, 3):
                for fast in FAST:
                    with ltr.Context(hfov=hfov, keyframe_batch=B, **FAST[fast]) as ctx:
                        got, _, _ = _run(ctx, m, xyzi, off, poses, inv, mode, alpha, 0.05)
                    if not np.array_equal(got, exp):
                        bad.append((mode, alpha, B, fast, np.flatnonzero(got != exp)[:5].tolist()))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------ 4. cull bound
def cull_scene(seed, coeff, n_tiles=600):
    """One keyframe whose scan returns fill every pixel at range s; 128-point patches (one tile each, radius <= 5 cm) at ranges
    around s (1 - c), within a few centimetres of the cull bound smax (1 - c) <= rmin - 1 mm: some tiles are culled, some are not and
    hold candidates, some hold none."""
    rng = np.random.default_rng(seed)
    alpha = 1.0                                                       # 50 x 360 pixels: the map has more points than the image pixels,
    rows, cols = ltr.reset_rimg_size(alpha)                           # which the pass requires before it culls
    s = F32(20.0)
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    az = np.deg2rad(c.ravel() * 360.0 / cols - 180.0); el = np.deg2rad((1.0 - r.ravel() / rows) * 50.0 - 25.0)
    d = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], 1)
    scan = np.concatenate([(d * s).astype(F32), np.zeros((len(d), 1), F32)], 1)
    tiles = []
    for _ in range(n_tiles):
        a0, e0 = rng.uniform(-np.pi * 0.95, np.pi * 0.95), np.deg2rad(rng.uniform(-20.0, 20.0))
        rho0 = float(s) * (1.0 - coeff) + rng.uniform(-0.08, 0.08)
        a = a0 + rng.uniform(-1.0, 1.0, 128) * 0.001; e = e0 + rng.uniform(-1.0, 1.0, 128) * 0.001
        rho = rho0 + rng.uniform(-0.02, 0.02, 128)
        tiles.append(np.stack([rho * np.cos(e) * np.cos(a), rho * np.cos(e) * np.sin(a), rho * np.sin(e)], 1))
    m = np.concatenate(tiles).astype(F32)
    return np.concatenate([m, np.ones((len(m), 1), F32)], 1), scan, np.array([0, len(scan)], np.int64), alpha


@pytest.mark.parametrize("coeff", [0.05, 0.2])
def test_cull_bound_is_sound(coeff):
    m, scan, off, alpha = cull_scene(21, coeff)
    I4 = np.eye(4)[None]
    exp = A.remove_pass(m, scan, off, I4, oracle.MODE_HD, alpha, coeff)
    assert 0 < exp.sum() < len(m)
    res = {}
    for fast in FAST:
        with ltr.Context(**FAST[fast]) as ctx:
            res[fast] = _run(ctx, m, scan, off, I4, I4, ltr.MODE_HD, alpha, coeff)
    for fast, (got, n, st) in res.items():
        assert np.array_equal(got, exp), (fast, np.flatnonzero(got != exp)[:8])
    culled = res[2][2][6]
    print(f"c = {coeff}: {int(exp.sum())} of {len(m)} flagged, {culled:.0f} pairs culled")
    assert 0 < culled < len(m)


# ------------------------------------------------------------------------------------------------------------ 5. kept scan images
@pytest.mark.parametrize("cache_mb", [None, "0"])
def test_kept_images_alternate_constant_and_adaptive(small_pair, small_maps, monkeypatch, cache_mb):
    if cache_mb is None:
        monkeypatch.delenv("LTR_SCAN_IMAGE_CACHE_MB", raising=False)
    else:
        monkeypatch.setenv("LTR_SCAN_IMAGE_CACHE_MB", cache_mb)
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)
    m = small_maps[0]
    calls = [None, 0.05, None, 0.2, 0.05, None, 0.05]   # None: the constant 0.1

    def one(ctx, mh, ss, ps, coeff):
        if coeff is None:
            ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)
        else:
            ctx.remove_pass_adaptive(mh, ss, ps, ltr.MODE_HD, 2.5, coeff)
        return ctx.flags_download(mh)

    fresh = {}
    for coeff in set(calls):
        with ltr.Context() as ctx:
            fresh[coeff] = one(ctx, ctx.cloud_upload(m), ctx.scanset_upload(c.xyzi, c.offsets), ctx.poses_upload(c.poses, inv), coeff)
    assert not np.array_equal(fresh[None], fresh[0.05])
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        for coeff in calls:
            assert np.array_equal(one(ctx, mh, ss, ps, coeff), fresh[coeff]), coeff
    assert np.array_equal(fresh[0.05], A.remove_pass(m, c.xyzi, c.offsets, inv, oracle.MODE_HD, 2.5, 0.05))


# ------------------------------------------------------------------------------------------------------------ 6. orchestrator
def test_orchestrator_applies_the_coefficient(small_pair):
    """Step 1's removeOnce(2.5) with the coefficient on: the pass log's count and the static map equal the restatement on the
    orchestrator's own map before the pass (partitioned, then octree-downsampled at 0.05 by the oracle); turning it off again gives the
    constant threshold's results."""
    c, q = small_pair
    res = {}
    for coeff in (0.05, 0.0):
        G = removert.Removerter(num_knn=2, knn_thr=0.01)
        G.set_adaptive_threshold(coeff)
        G.load_session(0, c.xyzi, c.offsets, c.poses, oracle.inverse_poses(c.poses))
        G.load_session(1, q.xyzi, q.offsets, q.poses, oracle.inverse_poses(q.poses))
        G.run_step0()
        G.stage("makeGlobalMap")
        M = G.cloud("map_global_curr_", 0)
        G.stage("removeHighDynamicPoints")
        log = G.log()
        res[coeff] = (M, log, G.cloud("map_global_curr_static_", 0))
        G.close()
    M, log, static = res[0.05]
    inv = oracle.inverse_poses(c.poses)
    flags = A.remove_pass(M, c.xyzi, c.offsets, inv, oracle.MODE_HD, 2.5, 0.05)
    assert log[0][0] == "removeOnce" and log[0][1] == len(M) and log[0][2] == int(flags.sum()), log[0]
    exp = oracle.voxel(M[flags == 0], 0.05)
    assert static.shape == exp.shape and np.array_equal(static.view(np.uint32), exp.view(np.uint32))
    M0, log0, static0 = res[0.0]
    const = oracle.remove_pass(M0, c.xyzi, c.offsets, inv, oracle.MODE_HD, 2.5)
    assert log0[0][2] == int(const.sum()) and log0[0][2] != log[0][2]


def test_orchestrator_rejects_bad_coefficients():
    with removert.Removerter() as G:
        for bad in (-0.05, 1.0, 1.5, float("nan"), float("inf")):
            with pytest.raises(Exception):
                G.set_adaptive_threshold(bad)
        G.set_adaptive_threshold(0.05)
        G.set_adaptive_threshold(0.0)


# ------------------------------------------------------------------------------------------------------------ 7. driver
SUMMARY = re.compile(r" Adaptive threshold: coefficient ([0-9.e+-]+)")


def _drive(tmp_path, tag, args, world=1):
    out = tmp_path / f"out_{tag}"
    cfg = tmp_path / f"params_{tag}.yaml"
    cfg.write_text(_PARAMS.format(out=out, d=tmp_path))
    logs = []
    procs = []
    for rank in range(world):
        e = dict(os.environ, RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), LTR_NCCL_ID_FILE=str(tmp_path / f"nccl_{tag}"))
        procs.append(subprocess.Popen([BIN, "--config", str(cfg)] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=e))
    for p in procs:
        o, _ = p.communicate(timeout=600)
        assert p.returncode == 0, o
        logs.append(o)
    return out, "".join(logs)


def test_driver_writes_what_the_orchestrator_holds(tmp_path, small_pair):
    _dataset(tmp_path, small_pair)
    out_plain, log_plain = _drive(tmp_path, "plain", [])
    out, log = _drive(tmp_path, "adaptive", ["--adaptive-threshold=0.05"])
    plain, adaptive = _tree(out_plain), _tree(out)
    assert set(plain) == set(adaptive), "the option must not change the output tree's layout"
    assert not SUMMARY.search(log_plain) and float(SUMMARY.search(log).group(1)) == pytest.approx(0.05)
    _, log_bare = _drive(tmp_path, "bare", ["--adaptive-threshold"])
    assert float(SUMMARY.search(log_bare).group(1)) == pytest.approx(0.05)
    c, q = small_pair
    kc = removert.parse_keyframes(c.K, 2, 5, 1)
    kq = removert.parse_keyframes_in_roi(q.poses, c.poses[kc], 1)
    G = removert.Removerter(num_knn=3, knn_thr=0.1)
    G.set_adaptive_threshold(0.05)
    for s, d, ks in ((0, c, kc), (1, q, kq)):
        xyzi = np.concatenate([d.scan(k) for k in ks])
        off = np.concatenate([[0], np.cumsum([len(d.scan(k)) for k in ks])])
        poses = removert.read_poses(str(tmp_path / ("central" if s == 0 else "query") / "poses.txt"))[ks]
        G.load_session_raw(s, xyzi, off, poses, removert.inverse_poses(poses))
    G.run_step0()
    G.run_step12()
    G.run_step3()
    compared = []
    for rel in adaptive:
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
    assert any(adaptive[k] != plain[k] for k in compared), "the coefficient changed nothing"
    G.close()


@pytest.mark.parametrize("value", ["0", "1", "1.5", "-0.05", "nan", "inf", "abc", "0.05x", ""])
def test_driver_bad_value_exits_2(tmp_path, value):
    r = subprocess.run([BIN, "--config", str(tmp_path / "unused.yaml"), "--adaptive-threshold=" + value], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2, r.stdout + r.stderr


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
def test_driver_two_ranks(tmp_path, small_pair):
    _dataset(tmp_path, small_pair)
    out1, _ = _drive(tmp_path, "one", ["--adaptive-threshold=0.05"])
    out2, _ = _drive(tmp_path, "two", ["--adaptive-threshold=0.05"], world=2)
    one, two = _tree(out1), _tree(out2)
    assert set(one) == set(two)
    for k in one:
        assert one[k] == two[k], k


# ------------------------------------------------------------------------------------------------------------ 8. ABI
def test_abi_rejects_bad_coefficients_and_returns_its_memory(small_pair, small_maps):
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(small_maps[0]); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        for bad in (0.0, -0.0, -0.05, 1.0, 2.0, float("nan"), float("inf"), float("-inf")):
            with pytest.raises(ltr.LtrError) as e:
                ctx.remove_pass_adaptive(mh, ss, ps, ltr.MODE_HD, 2.5, bad)
            assert e.value.code == -1, bad
        ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)            # the flag array of the map is allocated by its first pass
        ctx.scan_images_release(True)
        base = ctx.memory_stats()[0]
        for coeff in (0.05, 0.2):
            ctx.remove_pass_adaptive(mh, ss, ps, ltr.MODE_HD, 2.5, coeff)
            ctx.remove_pass_adaptive(mh, ss, ps, ltr.MODE_ND, 2.5, coeff)
        ctx.scan_images_release(True)
        assert ctx.memory_stats()[0] == base
