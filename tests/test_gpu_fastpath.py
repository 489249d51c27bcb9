"""The fast rejection path (project_fast.cuh) never changes a result.  Its margins are a DERIVED error bound (DESIGN.md section 4.1)
times a safety factor; here (1) the two arctangent polynomials are swept over EVERY float of their domain and must meet the error
constants the bound quotes, (2) measured deviations of whole projections from the reference arithmetic must stay below the derived
bound itself (margin / safety) on adversarial geometry, and (3) flags / visible points are identical with the fast path on and off."""
import numpy as np
import pytest

import oracle
import lt_mapper_b200 as ltr

pytestmark = pytest.mark.gpu


def _random_pose(rng, big=False):
    T = np.eye(4)
    q = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if np.linalg.det(q) < 0:
        q[:, 0] = -q[:, 0]
    T[:3, :3] = q
    T[:3, 3] = rng.uniform(-500, 500, 3) if big else rng.uniform(-60, 60, 3)
    return T


K_MARGIN_SAFETY = 1.5      # project_fast.cuh kMarginSafety
K_AZ_POLY_ERR = 6.8e-7     # project_fast.cuh kAzPolyErr
K_EL_POLY_ERR = 0.9e-7     # project_fast.cuh kElPolyErr


def _adversarial_world(rng, pose, n):
    """Points in the sensor frame with log-uniform range 0.5 .. 150 m, all directions, plus near-axis and near-seam sets, in the world frame."""
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    d[: n // 8, :2] *= 1e-3                                     # near the vertical axis (ill-conditioned azimuth)
    d[n // 8: n // 4, 1] = rng.uniform(-1e-4, 1e-4, n // 8); d[n // 8: n // 4, 0] = -np.abs(d[n // 8: n // 4, 0])   # azimuth seam +-pi
    r = np.exp(rng.uniform(np.log(0.5), np.log(150.0), n))[:, None]
    return ((d * r) @ pose[:3, :3].T + pose[:3, 3]).astype(np.float32)


def _certain(out, mg):
    """map_project_fast_kernel's certainty test on ltr_debug_fast_project's output (margins and seam limit of ltr_debug_margins)."""
    magic = np.float32(12582912.0)
    with np.errstate(invalid="ignore", over="ignore"):
        vcol, vrow = out[:, 0], out[:, 1]
        dc = np.abs(vcol - ((vcol + magic) - magic)); dr = np.abs(vrow - ((vrow + magic) - magic))
        lhs = (np.float64(mg[1]) * out[:, 3] + dc).astype(np.float32)
        return (lhs < np.float32(0.5) - mg[0]) & (dr < np.float32(0.5) - mg[2]) & (np.abs(out[:, 7]) < mg[8])


def _clamped(v_fast, v_ref, n):
    """Fast index (round half to even, the kernel's magic-number rounding) and reference index (std::round), both clamped to [0, n)."""
    with np.errstate(invalid="ignore"):
        return (np.clip(np.rint(v_fast.astype(np.float64)), 0, n - 1),
                np.clip(np.sign(v_ref) * np.floor(np.abs(v_ref.astype(np.float64)) + 0.5), 0, n - 1))


def _assert_certain_pixels_match(out, mg, rows, cols):
    """The statement the kernel relies on: a pair it calls certain has the reference's clamped column and row.  (A wrapped column
    distance hides a pair placed across the seam, and at hfov < 360 the two sides of the seam clamp to opposite edges.)"""
    c = _certain(out, mg)
    fc, ec = _clamped(out[:, 0], out[:, 4], cols)
    fr, er = _clamped(out[:, 1], out[:, 5], rows)
    assert not (c & (fc != ec)).any(), out[c & (fc != ec)][:3]
    assert not (c & (fr != er)).any(), out[c & (fr != er)][:3]
    return c


def test_atan_polynomials_exhaustive():
    """All 1 065 353 217 floats of [0, 1] through the azimuth polynomial and all 1 056 964 609 floats of [0, 0.5] through the short
    elevation polynomial, against atan() in double: the maxima must not exceed the constants of the error budget."""
    with ltr.Context() as ctx:
        e_az, a_az = ctx.debug_atan_sweep(0)
        e_el, a_el = ctx.debug_atan_sweep(1)
    print(f"azimuth polynomial: max |err| = {e_az:.3e} at a = {a_az!r};  elevation polynomial: max |err| = {e_el:.3e} at t = {a_el!r}")
    assert 0.0 < e_az <= K_AZ_POLY_ERR, (e_az, a_az)
    assert 0.0 < e_el <= K_EL_POLY_ERR, (e_el, a_el)


@pytest.mark.parametrize("alpha", [2.5, 3.0, 1.0])
def test_margins_dominate_measured_deviation(alpha):
    rng = np.random.default_rng(42)
    worst = np.zeros(3)
    with ltr.Context() as ctx:
        for trial in range(6):
            pose = _random_pose(rng, big=trial % 2 == 1)
            inv = np.linalg.inv(pose)
            world = _adversarial_world(rng, pose, 2_000_000)
            out, mg = ctx.debug_fast_project(world, inv, alpha)
            el_direct = bool(ctx.debug_margins(alpha)[5])
            ok = np.isfinite(out).all(axis=1)
            o = out[ok].astype(np.float64)
            rows, cols = ltr.reset_rimg_size(alpha)
            _assert_certain_pixels_match(out, ctx.debug_margins(alpha), rows, cols)
            # the error magnitude: at 360 degrees the seam wraps (the pixel itself is checked just above)
            dcol = np.abs(o[:, 0] - o[:, 4]); dcol = np.minimum(dcol, cols - dcol)
            m_col = mg[0] + mg[1] * o[:, 3]
            m_row = mg[2]
            m_r = mg[3] * o[:, 2] + 5e-6
            drow = np.abs(o[:, 1] - o[:, 5])
            if el_direct:
                # short elevation path: beyond |qz / rho| = 0.5 the fast elevation is clamped on purpose; there both pre-round rows must
                # lie at least a full pixel outside the image on the same side (-> the same clamped row), inside it the bound applies
                # classified by the REFERENCE's own elevation (its pre-round row), not by the generated coordinates: points a fraction of a
                # millimetre from the sensor move by more than that when the world coordinates are rounded to float
                ppr_r = rows * 180.0 / (np.pi * 50.0)
                el_ref = (0.5 * rows - o[:, 5]) / ppr_r
                inside = np.abs(el_ref) < np.arctan(0.4995)
                top = el_ref > np.arctan(0.5005)
                bot = el_ref < -np.arctan(0.5005)
                assert (o[top, 1] < -1.0).all() and (o[top, 5] < -1.0).all()
                assert (o[bot, 1] > rows).all() and (o[bot, 5] > rows).all()
                drow = drow[inside]
            worst = np.maximum(worst, [np.max(dcol / m_col), np.max(drow / m_row), np.max(np.abs(o[:, 2] - o[:, 6]) / m_r)])
            assert ok.mean() > 0.99
    print("max deviation / margin (col, row, range):", worst)
    # the margins are the derived bound x K_MARGIN_SAFETY: the measured deviation must stay below the DERIVED bound itself
    assert (worst * K_MARGIN_SAFETY < 1.0).all(), worst


@pytest.mark.parametrize("vfov,hfov", [(50.0, 360.0), (50.0, 359.0), (33.2, 180.0)])
def test_certain_pairs_keep_the_reference_pixel(vfov, hfov):
    """Every pair the certainty test calls certain has the reference's clamped column and row, on the adversarial geometry of the margin
    test and on points exactly on the seam of a keyframe turned by 90 degrees about z: there the fast sensor-frame y of a point below the
    sensor is -0 where the reference's is +0, so the fast azimuth is -pi and the reference's +pi."""
    rng = np.random.default_rng(43)
    quarter = np.eye(4); quarter[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]; quarter[:3, 3] = [3.25, -7.5, 1.125]
    quarter_inv = np.eye(4); quarter_inv[:3, :3] = quarter[:3, :3].T; quarter_inv[:3, 3] = -quarter[:3, :3].T @ quarter[:3, 3]
    n_seam = 4000
    el = rng.uniform(-1.4, 1.4, n_seam); r = rng.uniform(0.5, 100.0, n_seam)
    seam = np.stack([-r * np.cos(el), np.where(rng.random(n_seam) < 0.5, 0.0, -0.0), r * np.sin(el)], 1)   # azimuth exactly +-pi
    seam_world = (seam @ quarter[:3, :3].T + quarter[:3, 3]).astype(np.float32)
    with ltr.Context(vfov=vfov, hfov=hfov) as ctx:
        for alpha in (2.5, 1.0):
            rows, cols = ltr.reset_rimg_size(alpha, vfov, hfov)
            mg = ctx.debug_margins(alpha)
            for pose, inv, extra in ((_random_pose(rng), None, None), (_random_pose(rng, big=True), None, None), (quarter, quarter_inv, seam_world)):
                world = _adversarial_world(rng, pose, 500_000)
                if extra is not None:
                    world = np.concatenate([world, extra])
                out, _ = ctx.debug_fast_project(world, np.linalg.inv(pose) if inv is None else inv, alpha)
                c = _assert_certain_pixels_match(out, mg, rows, cols)
                assert c.mean() > 0.5


@pytest.mark.parametrize("mode,alpha", [(ltr.MODE_HD, 2.5), (ltr.MODE_HD, 1.0), (ltr.MODE_PD, 2.5), (ltr.MODE_ND, 2.5)])
def test_fast_path_equals_exact_path(small_pair, small_maps, mode, alpha):
    c = small_pair[0]
    m = small_maps[0] if mode == ltr.MODE_HD else small_maps[1][::5]
    inv = oracle.inverse_poses(c.poses)
    res = []
    for fast, cull in ((False, False), (True, False), (True, True)):
        with ltr.Context(fast_path=fast, cull=cull, keyframe_batch=3) as ctx:
            mh = ctx.cloud_upload(m)
            ss = ctx.scanset_upload(c.xyzi, c.offsets)
            ps = ctx.poses_upload(c.poses, inv)
            n = ctx.remove_pass(mh, ss, ps, mode, alpha)
            st = ctx.last_pass_stats()
            vis = ctx.parse_projected(mh, ps, 0, c.K, 3.0)
            st2 = ctx.last_pass_stats()
            res.append((n, ctx.flags_download(mh), ctx.scanset_download(vis), st, st2))
    for other in res[1:]:
        assert res[0][0] == other[0] and np.array_equal(res[0][1], other[1])
        assert np.array_equal(res[0][2][1], other[2][1]) and np.array_equal(res[0][2][0].view(np.uint32), other[2][0].view(np.uint32))
    exp = oracle.remove_pass(m, c.xyzi, c.offsets, inv, mode, alpha)
    assert np.array_equal(res[2][1], exp)
    st, st2 = res[2][3], res[2][4]
    print("culled share %.3f" % (st[6] / st[0]))
    if mode == ltr.MODE_ND:
        assert st[6] == 0         # never culled: a far point can still win its pixel
    print("remove pass: pairs %.3g exact-path share %.4f atomics %.3g | parse: exact-path share %.4f" % (st[0], st[2] / st[0], st[3], st2[2] / st2[0]))
    if mode == ltr.MODE_HD:
        assert st[2] / st[0] < 0.5


def test_fast_path_with_extrinsic_and_order(small_pair):
    """Non-identity LiDAR->base extrinsic (two-step transform) and the PCL>=1.10 summation order."""
    c = small_pair[0].subset(0, 3)
    l2b = np.eye(4)
    a = 0.05
    l2b[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
    l2b[:3, 3] = [0.3, -0.1, 0.2]
    inv = oracle.inverse_poses(c.poses)
    merged = np.concatenate([oracle.transform(oracle.transform(c.scan(k), l2b, 1), c.poses[k], 1) for k in range(c.K)])
    m = oracle.voxel(merged, 0.1)
    exp = oracle.remove_pass(m, c.xyzi, c.offsets, inv, oracle.MODE_HD, 2.5, lidar2base=l2b, order=1)
    e_vis, _ = oracle.parse_projected(m, inv[1], 3.0, lidar2base=l2b, order=1)
    for fast, cull in ((False, False), (True, False), (True, True)):
        with ltr.Context(lidar2base=l2b, base2lidar=oracle.inverse4x4(l2b), transform_order=1, fast_path=fast, cull=cull) as ctx:
            mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
            ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)
            assert np.array_equal(ctx.flags_download(mh), exp)
            pts, off = ctx.scanset_download(ctx.parse_projected(mh, ps, 1, 2, 3.0))
            assert np.array_equal(pts.view(np.uint32), e_vis.view(np.uint32))
            g = ctx.cloud_download(ctx.merge_scans_global(ss, ps))
            assert np.array_equal(g.view(np.uint32), merged.view(np.uint32))
    assert exp.sum() > 0


@pytest.mark.parametrize("vfov,hfov", [(40.0, 360.0), (33.2, 180.0), (90.0, 360.0), (50.0, 359.0)])
def test_non_default_fov(small_pair, small_maps, vfov, hfov):
    """sequence_vfov / sequence_hfov other than 50 x 360 (the oracle side of these is pinned against the compiled reference in
    tests/test_ref_pin.py): heavy row / column clamping at the narrow settings, every kernel variant."""
    c = small_pair[0]
    m = small_maps[0]
    inv = oracle.inverse_poses(c.poses)
    exp = {(mode, a): oracle.remove_pass(m, c.xyzi, c.offsets, inv, mode, a, 0.1, vfov=vfov, hfov=hfov)
           for mode in (oracle.MODE_HD, oracle.MODE_ND, oracle.MODE_PD) for a in (2.5, 0.7)}
    e_vis, _ = oracle.parse_projected(m, inv[2], 3.0, vfov=vfov, hfov=hfov)
    for fast, cull in ((False, False), (True, False), (True, True)):
        with ltr.Context(vfov=vfov, hfov=hfov, fast_path=fast, cull=cull) as ctx:
            mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
            for (mode, a), e in exp.items():
                ctx.remove_pass(mh, ss, ps, mode, a)
                assert np.array_equal(ctx.flags_download(mh), e), (fast, cull, mode, a)
            pts, off = ctx.scanset_download(ctx.parse_projected(mh, ps, 2, 3, 3.0))
            assert np.array_equal(pts.view(np.uint32), e_vis.view(np.uint32)), (fast, cull)
    assert all(e.sum() > 0 for e in exp.values())


@pytest.mark.parametrize("vfov,hfov", [(50.0, 360.0), (33.2, 180.0)])
def test_scan_range_image_fast_equals_exact(small_pair, vfov, hfov):
    """The scan range image itself (Removerter.cpp:109-156), fast pixel evaluation on and off, against the oracle (whose scan2RangeImg
    is pinned against the compiled reference): identical bits, at coarse and fine resolutions, with range ties and degenerate points."""
    c = small_pair[0]
    rng = np.random.default_rng(11)
    extra = np.array([[0, 0, 1, 0], [0, 0, -2, 0], [0, 0, 0, 0], [-5, 0.0, 0.3, 0], [-5, -0.0, 0.3, 0], [1e-20, 1e-20, 1e-20, 0], [3, 4, 0, 0], [3, 4, 0, 1]], np.float32)
    xyzi = np.concatenate([c.xyzi, c.scan(1)[::-1], rng.normal(0, 20, (50000, 4)).astype(np.float32), extra])
    off = np.array([0, c.offsets[3], len(xyzi)], np.int64)          # two ragged "keyframes"
    for fast in (False, True):
        with ltr.Context(vfov=vfov, hfov=hfov, fast_path=fast) as ctx:
            ss = ctx.scanset_upload(xyzi, off)
            for alpha in (0.5, 1.0, 2.5, 3.0):
                rows, cols = oracle.reset_rimg_size(alpha, vfov, hfov)
                for k in (0, 1):
                    exp = oracle.scan2rimg(xyzi[off[k]:off[k + 1]], rows, cols, vfov, hfov)
                    got = ctx.debug_scan_rimg(ss, k, alpha)
                    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)), (fast, alpha, k)

