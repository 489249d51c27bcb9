"""The azimuth seam in every unpadded variant of the fast map projection (project_fast.cuh).

Near azimuth +-pi the fast transform can give a sensor-frame y whose sign differs from the reference's: exactly when y is zero, or
within the transform error of zero.  The reference then takes the other side of the seam -- column 0 against C - 1 at 360 degrees, the
opposite clamped edge of the image otherwise -- although the fast column is far from a rounding boundary and looks certain.  The kernel
therefore never calls a pair certain whose fast azimuth is within half a pixel of +-pi (`FastCfg::az_seam_lim`).

These scenes put map points exactly there: keyframes rotated by quarter and half turns with exact 0 / +-1 entries and float32-exact translations,
rays at azimuth exactly +-pi and a few ulps off it, elevations across, above and below the field of view, map points in front of, on
and behind each scan return, and a competitor in the other seam pixel of the same row.  They run through the true-minimum variants
(ND pass, deferred and immediate; visible-point extraction in tile order and in map order) at every field of view, and through the
unpadded scan-minus-map variants (HD / PD at 90 x 360, 50 x 359 and 33.2 x 180), at keyframe batches 1, 3, 32 and across two launches,
with keyframes without fast constants and non-finite map points mixed in.  Flags and the bits of the visible points must equal the
oracle's and the all-exact kernel's.  The deferred mode's retry after a full candidate list runs in a child process with the list
shrunk by LTR_DEFERRED_LIST_CAP.

The tests without the gpu mark check on the CPU, with numpy copies of make_kf_fast and of the fast transform, that the scene really
contains seam points whose fast y has the other sign than the reference's.
"""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import oracle

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KNOB = "LTR_DEFERRED_LIST_CAP"

DEFAULT_FOV = (50.0, 360.0)
UNPADDED_FOVS = ((90.0, 360.0), (50.0, 359.0), (33.2, 180.0))   # general elevation path; unpadded short path (the seam clamps to opposite edges)
BATCHES = (1, 3, 32)
ND_ALPHA = 2.5
PARSE_ALPHAS = (3.0, 1.0)
CAND_ALPHAS = (2.5, 1.0)
THRES = 0.1


# ---------------------------------------------------------------------------------------------------------------- scene
# Keyframe k is rotated by ROTATIONS[k % 8]: quarter turns about z, then half a turn about x and two turns that swap axes.  All have exact
# 0 / +-1 entries, so that a point on the seam stays exactly on it.  Which of them flip the sign of a zero y depends on the signs of the
# zero terms of the fast FMA chain: here the 90-degree turn about z and the last one do it for points below the sensor (z < 0), the
# half turn about x and the seventh for points above it (test_selfcheck_fast_y_has_the_other_sign_on_the_seam).
ROTATIONS = [np.array(r, np.float64) for r in (
    [[1, 0, 0], [0, 1, 0], [0, 0, 1]], [[0, -1, 0], [1, 0, 0], [0, 0, 1]], [[-1, 0, 0], [0, -1, 0], [0, 0, 1]], [[0, 1, 0], [-1, 0, 0], [0, 0, 1]],
    [[1, 0, 0], [0, -1, 0], [0, 0, -1]], [[0, 0, 1], [0, 1, 0], [-1, 0, 0]], [[0, 0, -1], [1, 0, 0], [0, -1, 0]], [[1, 0, 0], [0, 0, 1], [0, -1, 0]])]


def _pose(k, t):
    p = np.eye(4)
    p[:3, :3] = ROTATIONS[k % len(ROTATIONS)]
    p[:3, 3] = t
    return p


def _sph(az, el, r):
    """Sensor-frame points; az = +-pi gives y = +-0.0 exactly."""
    az, el, r = np.broadcast_arrays(*(np.atleast_1d(np.asarray(v, np.float64)) for v in (az, el, r)))
    ce = np.cos(el)
    x, y, z = r * ce * np.cos(az), r * ce * np.sin(az), r * np.sin(el)
    y = np.where(np.abs(az) == np.pi, np.copysign(0.0, az), y)
    return np.stack([x, y, z], 1)


def _to_world(p_s, pose):
    return (p_s @ pose[:3, :3].T + pose[:3, 3]).astype(F32)


def _xyzi(p, i=1.0):
    return np.concatenate([np.asarray(p, F32).reshape(-1, 3), np.full((len(p), 1), i, F32)], 1)


SEAM_AZ = np.array([np.pi, -np.pi] + [s * (np.pi - j * 2.4e-7) for j in (1, 2, 3) for s in (1, -1)])   # +-pi and +-pi -+ 1..3 ulps of pi
COMPETITOR_OFF = 1.4e-3       # rad: inside the edge column at every alpha <= 3 and field of view used here


def seam_scene(seed, K, vfov=50.0, nonrigid=(), nonfinite=False):
    """(map xyzi, per-keyframe scans, poses, inverse poses, keyframe of each map point).  Per keyframe: rays on the seam at elevations
    across the field of view, just inside and outside its edges, and far above and below it (both signs of z), each with a scan return
    and a random non-empty subset of map points in front of it, on it and behind it; for each seam ray a nearer or farther competitor
    (with its own scan return) in the other seam pixel of the same row; and random rays elsewhere, so that every pass flags something."""
    rng = np.random.default_rng(seed)
    half = 0.5 * vfov
    els = np.deg2rad(np.concatenate([rng.uniform(-0.95 * half, 0.95 * half, 10), [0.0],
                                     np.array([0.99, 1.01, 1.2]) * half, -np.array([0.99, 1.01, 1.2]) * half,
                                     [26.0, 27.0, 45.0, 80.0], [-26.0, -27.0, -45.0, -80.0]]))
    poses, scans, mpts, owner = [], [], [], []
    for k in range(K):
        pose = _pose(k, np.round(rng.uniform(-20, 20, 3) * 64) / 64)   # float32-exact translation: seam points survive the round trip
        if k in nonrigid:
            pose[:3, :3] *= 1.0 + 1e-3 * (k + 1)             # ||A A^T - I|| >= 1e-5: this keyframe has no fast constants
        az_s = np.repeat(SEAM_AZ, len(els)); el_s = np.tile(els, len(SEAM_AZ))
        az_c = -np.sign(az_s) * (np.pi - COMPETITOR_OFF)
        az_r = rng.uniform(-np.pi * 0.97, np.pi * 0.97, 120); el_r = np.deg2rad(rng.uniform(-half, half, 120))
        az = np.concatenate([az_s, az_c, az_r]); el = np.concatenate([el_s, el_s, el_r])
        rs = rng.uniform(3.0, 60.0, len(az))
        scans.append(_xyzi(_sph(az, el, rs), 0.0))
        n_s = len(az_s)
        pts = []
        # seam and random rays: a random non-empty subset of {in front, on, behind}
        sub = np.r_[0:n_s, 2 * n_s:len(az)]
        pick = rng.integers(1, 8, len(sub))
        for bit, f in ((1, rng.uniform(0.3, 0.95, len(sub))), (2, 1.0 + rng.uniform(0.0, 0.004, len(sub))), (4, rng.uniform(1.05, 2.0, len(sub)))):
            sel = (pick & bit) != 0
            pts.append(_sph(az[sub][sel], el[sub][sel], (rs[sub] * f)[sel]))
        # competitors: nearer or farther than the seam ray's points, in the other seam pixel
        pts.append(_sph(az_c, el_s, rs[n_s:2 * n_s] * rng.uniform(0.2, 1.5, n_s)))
        p = np.concatenate(pts).astype(F32).astype(np.float64)
        mpts.append(_to_world(p, pose)); owner.append(np.full(len(p), k))
        poses.append(pose)
    poses = np.stack(poses)
    m, owner = np.concatenate(mpts), np.concatenate(owner)
    if nonfinite:
        bad = np.array([[np.nan, 1, 1], [1, np.nan, 1], [1, 1, np.nan], [np.inf, 0, 0], [-np.inf, 0, 0], [0, np.inf, 0], [0, -np.inf, 0],
                        [0, 0, np.inf], [0, 0, -np.inf], [np.inf, np.inf, 0], [-np.inf, np.inf, np.inf], [np.nan, np.nan, np.nan]], F32)
        at = rng.integers(0, len(m), len(bad))
        m = np.insert(m, at, bad, axis=0); owner = np.insert(owner, at, -1)
        m = np.concatenate([m, bad, bad[:5]]); owner = np.concatenate([owner, np.full(len(bad) + 5, -1)])
    return _xyzi(m), scans, poses, oracle.inverse_poses(poses), owner


def small_map(m, owner):
    """Fewer than 128 points (one partial tile: the visible-point extraction keeps map order): seam points of the keyframe rotated by 90
    degrees, plus the non-finite points if there are any."""
    sel = np.flatnonzero(owner == 1)[:110]
    return np.concatenate([m[sel], m[owner == -1][:6]])


def overflow_scene(seed=7, n_dup=300):
    """Three keyframes for launches of one: the first and the last have no fast constants (no list appends at all), the middle one
    sees a cluster of n_dup identical points alone in its pixel, which appends n_dup - 1 entries to the deferred candidate list."""
    m, scans, poses, inv, owner = seam_scene(seed, 3, nonrigid=(0, 2))
    cluster = _to_world(np.repeat(_sph(1.0, 0.1, 5.0), n_dup, 0).astype(F32).astype(np.float64), poses[1])
    m = np.concatenate([m, _xyzi(cluster)])
    return m, scans, poses, oracle.inverse_poses(poses)


def _scan_set(scans):
    return np.concatenate(scans), np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------- CPU copies
def kf_fast(inv_pose):
    """numpy copy of make_kf_fast (ltr_api.cu) for an identity extrinsic: A (3x3 f32), c_hi (3 f32), t_lo (3 f32), ok."""
    M = np.asarray(inv_pose, np.float64)[:3, :4]
    a, b, c, d, e, f, g, h, i = M[0, 0], M[0, 1], M[0, 2], M[1, 0], M[1, 1], M[1, 2], M[2, 0], M[2, 1], M[2, 2]
    det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g)
    ok = bool(np.isfinite(det) and 1e-6 < abs(det) < 1e6)
    for r1 in range(3):
        for r2 in range(r1, 3):
            dot = M[r1, 0] * M[r2, 0] + M[r1, 1] * M[r2, 1] + M[r1, 2] * M[r2, 2]
            ok = ok and abs(dot - (1.0 if r1 == r2 else 0.0)) < 1e-5
    adj = [(e * i - f * h), (c * h - b * i), (b * f - c * e), (f * g - d * i), (a * i - c * g), (c * d - a * f), (d * h - e * g), (b * g - a * h), (a * e - b * d)]
    cc = [-(adj[3 * r] * M[0, 3] + adj[3 * r + 1] * M[1, 3] + adj[3 * r + 2] * M[2, 3]) / det if ok else 0.0 for r in range(3)]
    A = M[:, :3].astype(F32)
    chi = np.array(cc).astype(F32)
    clo = [cc[r] - float(chi[r]) for r in range(3)]
    tlo = np.array([M[r, 0] * clo[0] + M[r, 1] * clo[1] + M[r, 2] * clo[2] for r in range(3)]).astype(F32)
    return A, chi, tlo, ok


def _fma_exact01(a, b, c):
    """fmaf(a, b, c) for a in {0, +-1}: the product is exact, the f64 sum of two floats is exact, one rounding to f32 (zero signs as IEEE)."""
    return (np.float64(a) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def fast_qy(p, inv_pose):
    """The fast path's sensor-frame y (fast_project): three chained FMAs on p - c_hi, started at -t_lo."""
    A, chi, tlo, ok = kf_fast(inv_pose)
    assert ok and np.isin(A, (-1.0, 0.0, 1.0)).all()
    dx, dy, dz = (p[:, j].astype(F32) - chi[j] for j in range(3))
    q = _fma_exact01(A[1, 0], dx, np.full(len(p), -tlo[1], F32))
    q = _fma_exact01(A[1, 1], dy, q)
    return _fma_exact01(A[1, 2], dz, q)


def ref_xyz(p, inv_pose):
    """transform_point (order 0): the double transform, rounded once to f32 (ref_math.cuh)."""
    m = np.asarray(inv_pose, np.float64)
    x, y, z = (p[:, j].astype(np.float64) for j in range(3))
    return [((((m[r, 0] * x) + (m[r, 1] * y)) + (m[r, 2] * z)) + m[r, 3]).astype(F32) for r in range(3)]


def seam_flips(m, owner, inv, K, nonrigid=()):
    """Per rigid keyframe: (sign of the point's z, count) of its own map points behind the sensor (x < 0, so the azimuth is near +-pi)
    whose fast y has the other sign bit than the reference's y."""
    out = {}
    for k in range(K):
        if k in nonrigid:
            continue
        sel = owner == k
        x, y, z = ref_xyz(m[sel, :3], inv[k])
        qy = fast_qy(m[sel, :3], inv[k])
        flip = (x < 0) & (np.signbit(qy) != np.signbit(y)) & (np.abs(y) < 1e-4 * np.abs(x))
        out[k] = (int((flip & (z > 0)).sum()), int((flip & (z < 0)).sum()))
    return out


# ---------------------------------------------------------------------------------------------------------------- column helpers
def certain(out, mg, seam_rule=True):
    """The kernel's certainty test on ltr_debug_fast_project's output: both pre-round coordinates farther than their margin from a
    rounding boundary and (seam_rule) the fast azimuth short of ltr_debug_margins' seam limit.  NaN is never certain."""
    magic = F32(12582912.0)
    with np.errstate(invalid="ignore", over="ignore"):
        vcol, vrow = out[:, 0].astype(F32), out[:, 1].astype(F32)
        dc = np.abs(vcol - ((vcol + magic) - magic))
        dr = np.abs(vrow - ((vrow + magic) - magic))
        lhs = (np.float64(mg[1]) * out[:, 3].astype(np.float64) + dc.astype(np.float64)).astype(F32)   # fmaf(m_col_b, r / rho, dc)
        c = (lhs < F32(0.5) - F32(mg[0])) & (dr < F32(0.5) - F32(mg[2]))
        if seam_rule:
            c &= np.abs(out[:, 7]) < F32(mg[8])
    return c


def clamped(v_f, v_e, n):
    """(fast index: round half to even, as the magic-number rounding; reference index: std::round, half away), both clamped to [0, n)."""
    with np.errstate(invalid="ignore"):
        v_f, v_e = v_f.astype(np.float64), v_e.astype(np.float64)
        fast = np.clip(np.rint(v_f), 0, n - 1)
        ref = np.clip(np.sign(v_e) * np.floor(np.abs(v_e) + 0.5), 0, n - 1)
    return fast, ref


def clamped_columns(out, cols):
    return clamped(out[:, 0], out[:, 4], cols)


def reach(ctx, m, inv, K, alpha, vfov, hfov, nonrigid=()):
    """Per rigid keyframe: pairs the margins alone call certain whose clamped fast column is not the reference's."""
    import lt_mapper_b200 as ltr
    _, cols = ltr.reset_rimg_size(alpha, vfov, hfov)
    mg = ctx.debug_margins(alpha)
    fin = np.isfinite(m[:, :3]).all(1)
    n = {}
    for k in range(K):
        if k in nonrigid:
            continue
        out, _ = ctx.debug_fast_project(m[fin, :3], inv[k], alpha)
        fast, ref = clamped_columns(out, cols)
        n[k] = int((certain(out, mg, seam_rule=False) & (fast != ref)).sum())
    return n


# ---------------------------------------------------------------------------------------------------------------- GPU checks
def _expect_true_min(m, scans, inv, vfov, hfov, small):
    xyzi, off = _scan_set(scans)
    fin = np.isfinite(m[:, :3]).all(1)
    nd = np.zeros(len(m), np.uint8)
    nd[fin] = oracle.remove_pass(m[fin], xyzi, off, inv, oracle.MODE_ND, ND_ALPHA, THRES, vfov=vfov, hfov=hfov)
    vis = {}
    for name, mm in (("map", m), ("small", small)):
        f = np.isfinite(mm[:, :3]).all(1)
        for a in PARSE_ALPHAS:
            vis[name, a] = [oracle.parse_projected(mm[f], inv[k], a, vfov=vfov, hfov=hfov)[0] for k in range(len(inv))]
    return nd, vis


def check_true_min(m, scans, poses, inv, small, vfov, hfov, batches):
    """Every case runs; the assertion lists all that differ from the oracle."""
    import lt_mapper_b200 as ltr
    nd, vis = _expect_true_min(m, scans, inv, vfov, hfov, small)
    assert nd.sum() > 0 and all(sum(len(v) for v in vs) > 0 for vs in vis.values())
    xyzi, off = _scan_set(scans)
    K = len(poses)
    bad = []
    for B in batches:
        for fast in (False, True):
            with ltr.Context(vfov=vfov, hfov=hfov, fast_path=fast, keyframe_batch=B) as ctx:
                mh, sh = ctx.cloud_upload(m), ctx.cloud_upload(small)
                ss = ctx.scanset_upload(xyzi, off); ps = ctx.poses_upload(poses, inv)
                ctx.remove_pass(mh, ss, ps, ltr.MODE_ND, ND_ALPHA, diff_thres=THRES)                 # deferred true minimum
                got = ctx.flags_download(mh)
                if not np.array_equal(got, nd):
                    bad.append(("ND deferred", B, fast, np.flatnonzero(got != nd)[:5].tolist()))
                ctx.flags_upload(mh, np.zeros(len(m), np.uint8))                                    # sharded: immediate true minimum
                for k0, k1 in ((0, K // 2), (K // 2, K)):
                    ctx.remove_pass(mh, ss, ps, ltr.MODE_ND, ND_ALPHA, diff_thres=THRES, kf_begin=k0, kf_end=k1, accumulate=True)
                got = ctx.flags_download(mh)
                if not np.array_equal(got, nd):
                    bad.append(("ND immediate", B, fast, np.flatnonzero(got != nd)[:5].tolist()))
                for (name, a), e in vis.items():
                    pts, o = ctx.scanset_download(ctx.parse_projected(mh if name == "map" else sh, ps, 0, K, a))
                    diff = [k for k in range(K) if not np.array_equal(pts[o[k]:o[k + 1]].view(np.uint32), e[k].view(np.uint32))]
                    if diff:
                        bad.append(("visible points", name, a, B, fast, diff))
    assert not bad, bad


def check_candidates(m, scans, poses, inv, vfov, hfov, batches):
    import lt_mapper_b200 as ltr
    xyzi, off = _scan_set(scans)
    fin = np.isfinite(m[:, :3]).all(1)
    exp = {}
    for mode, om in ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_PD, oracle.MODE_PD)):
        for a in CAND_ALPHAS:
            e = np.zeros(len(m), np.uint8)
            e[fin] = oracle.remove_pass(m[fin], xyzi, off, inv, om, a, THRES, vfov=vfov, hfov=hfov)
            exp[mode, a] = e
    assert all(e.sum() > 0 for e in exp.values())
    bad = []
    for B in batches:
        for fast, cull in ((False, False), (True, False), (True, True)):
            with ltr.Context(vfov=vfov, hfov=hfov, fast_path=fast, cull=cull, keyframe_batch=B) as ctx:
                mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(xyzi, off); ps = ctx.poses_upload(poses, inv)
                for (mode, a), e in exp.items():
                    ctx.remove_pass(mh, ss, ps, mode, a, diff_thres=THRES)
                    got = ctx.flags_download(mh)
                    if not np.array_equal(got, e):
                        bad.append(("HD" if mode == ltr.MODE_HD else "PD", a, B, fast, cull, np.flatnonzero(got != e)[:5].tolist()))
    assert not bad, bad


NONRIGID = (5,)


@pytest.mark.gpu
@pytest.mark.parametrize("vfov,hfov", (DEFAULT_FOV,) + UNPADDED_FOVS)
def test_seam_scene_reaches_the_flip(vfov, hfov):
    """The scene is worth testing: in keyframes of more than one rotation, pairs that the margins alone call certain have a clamped fast
    column that is not the reference's -- exactly the pairs the seam rule must take away from the fast path."""
    import lt_mapper_b200 as ltr
    m, scans, poses, inv, owner = seam_scene(1, 8, vfov, nonrigid=NONRIGID)
    with ltr.Context(vfov=vfov, hfov=hfov) as ctx:
        for a in (ND_ALPHA,) + PARSE_ALPHAS:
            n = reach(ctx, m, inv, len(poses), a, vfov, hfov, NONRIGID)
            print(f"fov {vfov} x {hfov}, alpha {a}: certain pairs with the other column, per keyframe: {n}")
            rows, cols = ltr.reset_rimg_size(a, vfov, hfov)
            seam_col = 0.5 * cols - np.pi * cols * 180.0 / (np.pi * hfov)    # pre-round column of azimuth -pi
            if abs(abs(seam_col - np.round(seam_col)) - 0.5) < 0.01:
                continue        # on a rounding boundary (50 x 359 at alpha 1 and 3): no pair there is certain, so none can be misplaced
            assert len({k % 8 for k, v in n.items() if v > 0}) >= 2, n


@pytest.mark.gpu
@pytest.mark.parametrize("vfov,hfov", (DEFAULT_FOV,) + UNPADDED_FOVS)
def test_certain_pairs_keep_the_reference_column(vfov, hfov):
    """The statement the kernel relies on: every pair its certainty test (margins and seam rule) calls certain has the reference's
    clamped column and row."""
    import lt_mapper_b200 as ltr
    m, scans, poses, inv, owner = seam_scene(2, 8, vfov, nonrigid=NONRIGID)
    fin = np.isfinite(m[:, :3]).all(1)
    with ltr.Context(vfov=vfov, hfov=hfov) as ctx:
        for a in (ND_ALPHA,) + PARSE_ALPHAS:
            rows, cols = ltr.reset_rimg_size(a, vfov, hfov)
            mg = ctx.debug_margins(a)
            for k in range(len(poses)):
                if k in NONRIGID:
                    continue
                out, _ = ctx.debug_fast_project(m[fin, :3], inv[k], a)
                c = certain(out, mg)
                fast, ref = clamped_columns(out, cols)
                bad = c & (fast != ref)
                assert not bad.any(), (a, k, out[bad][:3])
                fr, er = clamped(out[:, 1], out[:, 5], rows)
                assert not (c & (fr != er)).any(), (a, k)
                assert c.mean() > 0.5


@pytest.mark.gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("vfov,hfov", (DEFAULT_FOV,) + UNPADDED_FOVS)
def test_true_minimum_variants_at_the_seam(vfov, hfov, B):
    """ND pass (deferred, and sharded over two calls that accumulate: the immediate mode) and the visible-point extraction (a map of
    >= 128 points: near-to-far tile order; one of < 128: map order) at alpha 3.0 and 1.0."""
    m, scans, poses, inv, owner = seam_scene(3, 8, vfov, nonrigid=NONRIGID, nonfinite=True)
    check_true_min(m, scans, poses, inv, small_map(m, owner), vfov, hfov, (B,))


@pytest.mark.gpu
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("vfov,hfov", UNPADDED_FOVS)
def test_unpadded_candidate_variants_at_the_seam(vfov, hfov, B):
    """HD and PD where the guard-padded test image does not apply: the general elevation path (90 x 360) and a field of view short of
    360 degrees, where the two sides of the seam clamp to opposite edges of the image."""
    m, scans, poses, inv, owner = seam_scene(4, 8, vfov, nonrigid=NONRIGID, nonfinite=True)
    check_candidates(m, scans, poses, inv, vfov, hfov, (B,))


@pytest.mark.gpu
def test_thirty_six_keyframes_at_the_seam():
    """More keyframes than one launch of 32 (32 + 4), with a keyframe without fast constants in the second launch."""
    m, scans, poses, inv, owner = seam_scene(5, 36, nonrigid=(5, 33), nonfinite=True)
    check_true_min(m, scans, poses, inv, small_map(m, owner), *DEFAULT_FOV, (32,))
    m, scans, poses, inv, owner = seam_scene(6, 36, 50.0, nonrigid=(5, 33), nonfinite=True)
    check_candidates(m, scans, poses, inv, 50.0, 359.0, (32,))


@pytest.mark.gpu
@pytest.mark.parametrize("vfov,hfov", (DEFAULT_FOV, (50.0, 359.0)))
def test_pairs_within_half_a_pixel_of_the_seam_take_the_full_exact_path(vfov, hfov):
    """The seam band is half a pixel wide in every unpadded variant.  128 map points (one tile) 0.41-0.49 px of azimuth short of +-pi, with
    the offset chosen per side so that the column is far from a rounding boundary, at the centre of a row: the margins alone would settle
    them; the seam rule sends each through the full reference arithmetic (pass statistics [5]).  A band narrower by a tenth of a pixel
    would leave them on the fast path.  (It could not change a result: a pair whose fast y has the other sign is within its column
    margin of +-pi, and a certain pair's margin is far below a tenth of a pixel.  This checks the band as documented.)"""
    import lt_mapper_b200 as ltr
    a = 2.5
    rows, cols = ltr.reset_rimg_size(a, vfov, hfov)
    cs = cols * 180.0 / (np.pi * hfov)
    r_idx = 8 + (np.arange(64) * (rows - 16)) // 64
    el = np.deg2rad(((1.0 - r_idx / rows) * vfov - 0.5 * vfov))             # row centres: vrow = r up to rounding
    offs = np.linspace(0.41, 0.49, 81)
    az = []
    for s in (1.0, -1.0):
        seam_col = 0.5 * cols + s * np.pi * cs                                # pre-round column of azimuth s * pi
        frac = np.mod(seam_col - s * offs, 1.0)
        o = offs[np.argmax(np.abs(frac - 0.5))]                               # the offset whose column is farthest from a boundary
        az.append(np.full(len(el), s * (np.pi - o / cs)))
    az = np.concatenate(az)
    el = np.concatenate([el, el])
    p = _xyzi(_sph(az, el, np.full(len(az), 20.0)).astype(F32))
    assert len(p) == 128
    I4 = np.eye(4)[None]
    with ltr.Context(vfov=vfov, hfov=hfov) as ctx:
        out, _ = ctx.debug_fast_project(p[:, :3], I4[0], a)
        mg = ctx.debug_margins(a)
        assert certain(out, mg, seam_rule=False).all()                       # the margins alone would settle them
        assert not certain(out, mg).any()
        mh = ctx.cloud_upload(p); ps = ctx.poses_upload(I4, I4)
        ss = ctx.scanset_upload(_xyzi(p[:, :3] * 1.5, 0.0), [0, len(p)])
        ctx.remove_pass(mh, ss, ps, ltr.MODE_ND, a)
        assert ctx.last_pass_stats()[5] == len(p)
        pts, o = ctx.scanset_download(ctx.parse_projected(mh, ps, 0, 1, a))
        assert ctx.last_pass_stats()[5] == len(p)
        ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, a)
        if hfov != 360.0:                                                    # at 360 degrees HD takes the guard-padded variant
            assert ctx.last_pass_stats()[5] == len(p)
    e, _ = oracle.parse_projected(p, I4[0], a, vfov=vfov, hfov=hfov)
    assert np.array_equal(pts.view(np.uint32), e.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------- overflow retry
OVERFLOW_CHILD = textwrap.dedent("""
    import json, os, sys
    sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
    import numpy as np
    import oracle
    import lt_mapper_b200 as ltr
    import test_gpu_project_seam as T
    cap = {cap}
    m, scans, poses, inv = T.overflow_scene()
    xyzi, off = T._scan_set(scans)
    K = len(poses)
    nd = oracle.remove_pass(m, xyzi, off, inv, oracle.MODE_ND, T.ND_ALPHA, T.THRES)
    vis = [oracle.parse_projected(m, inv[k], 3.0)[0] for k in range(K)]
    res = {{}}
    with ltr.Context(keyframe_batch=1) as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(xyzi, off); ps = ctx.poses_upload(poses, inv)

        def run():
            l0 = ctx.kernel_launches()
            ctx.remove_pass(mh, ss, ps, ltr.MODE_ND, T.ND_ALPHA, diff_thres=T.THRES)
            flags = ctx.flags_download(mh)
            l1 = ctx.kernel_launches()
            h = ctx.parse_projected(mh, ps, 0, K, 3.0)
            pts, o = ctx.scanset_download(h)
            ctx.scanset_free(h)
            return flags, pts, o, l1 - l0, ctx.kernel_launches() - l1

        def check(flags, pts, o):
            assert np.array_equal(flags, nd), np.flatnonzero(flags != nd)[:10]
            for k in range(K):
                assert np.array_equal(pts[o[k]:o[k + 1]].view(np.uint32), vis[k].view(np.uint32)), k

        os.environ.pop({knob!r}, None)
        run()                                               # the first pass on the map allocates its flag array, which stays
        # list appends per launch with the full list: the first and last launch append nothing, the second more than the capacity
        appends = []
        for k in range(K):
            ctx.parse_projected(mh, ps, k, k + 1, 3.0)
            st = ctx.last_pass_stats()
            appends.append(st[2] - st[5])
        assert appends[0] <= cap < appends[1] and appends[2] <= cap, appends
        base = ctx.memory_stats()[0]
        flags, pts, o, nd_plain, parse_plain = run()
        check(flags, pts, o)
        assert ctx.memory_stats()[0] == base
        os.environ[{knob!r}] = str(cap)
        for _ in range(2):
            flags, pts, o, nd_small, parse_small = run()
            check(flags, pts, o)
            assert ctx.memory_stats()[0] == base, "the retry leaked scratch or the first output"
        res = dict(appends=appends, nd=[nd_plain, nd_small], parse=[parse_plain, parse_small])
    print("overflow " + json.dumps(res))
""")


@pytest.mark.gpu
def test_deferred_list_overflow_repeats_the_call_in_the_immediate_mode():
    """LTR_DEFERRED_LIST_CAP shrinks the deferred candidate list so that it overflows in the second of three launches and not in the
    first or third: the ND pass and the visible-point extraction must notice the sticky flag, free what the first attempt made, repeat
    the call in the immediate mode and return the oracle's result.  The repeat shows in the kernel-launch count, which a knob that is
    ignored would leave unchanged.  Runs in a child process so that the variable cannot reach other tests."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", OVERFLOW_CHILD.format(root=ROOT, cap=64, knob=KNOB)]
    env = {k: v for k, v in os.environ.items() if k != KNOB}
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    res = json.loads(r.stdout.split("overflow ", 1)[1])
    print(res)
    assert res["nd"][1] > res["nd"][0] and res["parse"][1] > res["parse"][0], res


# ---------------------------------------------------------------------------------------------------------------- CPU self-checks
def test_selfcheck_fast_y_has_the_other_sign_on_the_seam():
    """numpy copies of make_kf_fast and the three-FMA y of fast_project against the reference's double transform: the seam scene has
    points whose fast y has the other sign bit, in more than one rotation and with both signs of z."""
    for vfov in (50.0, 90.0, 33.2):
        m, scans, poses, inv, owner = seam_scene(1, 8, vfov, nonrigid=NONRIGID)
        flips = seam_flips(m, owner, inv, 8, NONRIGID)
        print(vfov, flips)
        assert len({k % 8 for k, (a, b) in flips.items() if a + b > 0}) >= 2, flips
        assert sum(a for a, _ in flips.values()) > 0 and sum(b for _, b in flips.values()) > 0, flips


def test_selfcheck_kf_fast_copy_is_exact_for_quarter_turns():
    """For these poses the constants are exact: A = R^T with 0 / +-1 entries, c_hi = the translation, t_lo = 0; the non-rigid keyframes
    have no fast constants."""
    m, scans, poses, inv, owner = seam_scene(1, 8, nonrigid=NONRIGID)
    for k in range(8):
        A, chi, tlo, ok = kf_fast(inv[k])
        assert ok == (k not in NONRIGID)
        if ok:
            assert np.array_equal(A.astype(np.float64), poses[k][:3, :3].T) and np.array_equal(chi.astype(np.float64), poses[k][:3, 3])
            assert not tlo.any()


def test_selfcheck_scene_shapes():
    """Map sizes on both sides of one 128-point tile, non-finite points where asked for, and the overflow scene's rigid middle keyframe."""
    m, scans, poses, inv, owner = seam_scene(3, 8, nonrigid=NONRIGID, nonfinite=True)
    assert len(m) >= 128 and 100 <= len(small_map(m, owner)) < 128
    assert (~np.isfinite(m[:, :3]).all(1)).sum() == 29 and (~np.isfinite(small_map(m, owner)[:, :3]).all(1)).sum() == 6
    m, scans, poses, inv = overflow_scene()
    assert [kf_fast(inv[k])[3] for k in range(3)] == [False, True, False]
    assert (m[-300:] == m[-1]).all()
