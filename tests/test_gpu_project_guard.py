"""The scan-minus-map projection gathers from a guard-padded test image: rows above and below the image replicate the rows the reference
clamps to, and one guard column follows the last, so the short elevation path needs no index clamp.  Column 0 and the guard column hold a
sentinel that sends their pairs to the full exact path (next to the seam the reference may choose the other side).  These scenes put pairs exactly where
that matters -- azimuth +-pi (the guard column), elevations between vfov/2 and beyond atan(0.5) (the guard rows), non-finite map points
(whose index must still stay inside the image), keyframes without fast constants mixed with rigid ones, and 128-point tiles whose pixel
rectangle touches the image border, the seam or the edge of an occluder (tile culling) -- at keyframe batches 1, 3 and 32.  Every HD and
PD pass must flag exactly what the all-exact kernel and the oracle flag."""
import numpy as np
import pytest

import oracle
import lt_mapper_b200 as ltr

pytestmark = pytest.mark.gpu

MODES = ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_PD, oracle.MODE_PD))
BATCHES = (1, 3, 32)


def _pose(rot_quarters, t):
    """Rotation about z by a multiple of 90 degrees with exact 0 / +-1 entries, so that a point on the seam stays exactly on it."""
    c, s = [(1, 0), (0, 1), (-1, 0), (0, -1)][rot_quarters % 4]
    p = np.eye(4)
    p[:3, :3] = [[c, -s, 0], [s, c, 0], [0, 0, 1]]
    p[:3, 3] = t
    return p


def _sph(az, el, r):
    """Sensor-frame points; az = +-pi gives y = +-0.0 exactly."""
    ce = np.cos(el)
    x, y, z = r * ce * np.cos(az), r * ce * np.sin(az), r * np.sin(el)
    y = np.where(np.abs(az) == np.pi, np.copysign(0.0, az), y)
    return np.stack([x, y, z], 1)


def _to_world(p_s, pose):
    return (p_s @ pose[:3, :3].T + pose[:3, 3]).astype(np.float32)


def _xyzi(p, i=1.0):
    return np.concatenate([np.asarray(p, np.float32), np.full((len(p), 1), i, np.float32)], 1)


def _check(m, scans, poses, inv, alpha, thres=0.1, batches=BATCHES, culled_min=None):
    xyzi = np.concatenate(scans) if sum(map(len, scans)) else np.zeros((0, 4), np.float32)
    off = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
    # the oracle restates the reference, whose pixel index of a non-finite point is undefined behaviour: it gets the finite points only.
    # A non-finite point has a NaN or infinite range, so scan - range > thres is false: it is never flagged and never wins a pixel.
    fin = np.isfinite(m[:, :3]).all(1)
    exp = []
    for _, om in MODES:
        e = np.zeros(len(m), np.uint8)
        e[fin] = oracle.remove_pass(m[fin], xyzi, off, inv, om, alpha, thres)
        exp.append(e)
    assert exp[0].sum() > 0, "the scene must flag something"
    culled = 0.0
    for B in batches:
        for fast, cull in ((False, False), (True, False), (True, True)):
            with ltr.Context(fast_path=fast, cull=cull, keyframe_batch=B) as ctx:
                mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(xyzi, off); ps = ctx.poses_upload(poses, inv)
                for (mode, _), e in zip(MODES, exp):
                    ctx.remove_pass(mh, ss, ps, mode, alpha, diff_thres=thres)
                    got = ctx.flags_download(mh)
                    assert np.array_equal(got, e), (B, fast, cull, mode, np.flatnonzero(got != e)[:10])
                    if cull:
                        st = ctx.last_pass_stats(); culled = max(culled, st[6] / max(st[0], 1.0))
    if culled_min is not None:
        assert culled >= culled_min, culled
    return exp


def _seam_and_rows_scene(rng, K, alpha, far_point=False, nonfinite=False, nonrigid=()):
    """Per keyframe: rays on the seam (azimuth exactly +-pi, and +-pi -+ a few ulps) and at steep elevations (between vfov/2 = 25 deg and
    far beyond atan(0.5) = 26.57 deg, up and down) with a scan return each; map points on the same rays in front of the return
    (candidates), just behind it and far behind it.  The scans are sparse, so most pixels next to a return are empty: a guard that
    replicated the wrong pixel would read "no return" there instead of the return."""
    poses, scans, mpts = [], [], []
    for k in range(K):
        pose = _pose(k, np.round(rng.uniform(-20, 20, 3) * 64) / 64)   # float32-exact translation: seam points survive the round trip
        if k in nonrigid:
            pose[:3, :3] *= 1.0 + 1e-3 * (k + 1)             # ||A A^T - I|| >= 1e-5: this keyframe has no fast constants
        els = np.concatenate([np.deg2rad(rng.uniform(-24, 24, 40)), np.deg2rad([25.0, 26.0, 26.6, 27.0, 30.0, 45.0, 60.0, 80.0, 89.0]),
                              -np.deg2rad([25.0, 26.0, 26.6, 27.0, 30.0, 45.0, 60.0, 80.0, 89.0])])
        seam = np.array([np.pi, -np.pi, np.nextafter(np.float32(np.pi), 0), -np.nextafter(np.float32(np.pi), 0)], np.float64)
        az_seam = np.repeat(seam, len(els)); el_seam = np.tile(els, len(seam))
        az_steep = rng.uniform(-np.pi * 0.98, np.pi * 0.98, 300)
        el_steep = np.deg2rad(rng.choice([1, -1], 300) * rng.uniform(24.0, 89.0, 300))
        az = np.concatenate([az_seam, az_steep]); el = np.concatenate([el_seam, el_steep])
        rs = rng.uniform(3.0, 60.0, len(az))
        scans.append(_xyzi(_sph(az, el, rs), 0.0))
        for f in (rng.uniform(0.3, 0.95, len(az)), 1.0 + rng.uniform(0.0, 0.004, len(az)), rng.uniform(1.05, 2.0, len(az))):
            mpts.append(_to_world(_sph(az, el, rs * f).astype(np.float32).astype(np.float64), pose))
        poses.append(pose)
    poses = np.stack(poses)
    m = np.concatenate(mpts)
    if far_point:                                            # a map point 8 km away: pixels without a return are not -inf in the test image
        m = np.concatenate([m, [[8000.0, 0.0, 0.0]]]).astype(np.float32)
    if nonfinite:
        bad = np.array([[np.nan, 1, 1], [1, np.nan, 1], [1, 1, np.nan], [np.inf, 0, 0], [-np.inf, 0, 0], [0, np.inf, 0], [0, -np.inf, 0],
                        [0, 0, np.inf], [0, 0, -np.inf], [np.inf, np.inf, 0], [-np.inf, np.inf, np.inf], [np.nan, np.nan, np.nan]], np.float32)
        m = np.insert(m, rng.integers(0, len(m), len(bad)), bad, axis=0)     # inside tiles of finite points
        m = np.concatenate([m, bad, bad[:5]])                                  # and a tile of their own
    return _xyzi(m), scans, poses, oracle.inverse_poses(poses)


@pytest.mark.parametrize("alpha", [2.5, 1.0, 3.0, 0.95 * 2.0])
def test_seam_and_guard_rows(alpha):
    m, scans, poses, inv = _seam_and_rows_scene(np.random.default_rng(11), 5, alpha)
    _check(m, scans, poses, inv, alpha)


def test_seam_and_guard_rows_without_the_empty_pixel_shortcut():
    m, scans, poses, inv = _seam_and_rows_scene(np.random.default_rng(12), 4, 2.0, far_point=True)
    _check(m, scans, poses, inv, 2.0)


@pytest.mark.parametrize("alpha", [2.5, 1.5])
def test_non_finite_map_points(alpha):
    m, scans, poses, inv = _seam_and_rows_scene(np.random.default_rng(13), 4, alpha, nonfinite=True)
    _check(m, scans, poses, inv, alpha)


def test_keyframes_with_and_without_fast_constants_in_one_batch():
    m, scans, poses, inv = _seam_and_rows_scene(np.random.default_rng(14), 7, 2.5, nonrigid=(1, 4, 5))
    _check(m, scans, poses, inv, 2.5)


def test_thirty_six_keyframes_across_batches():
    """More keyframes than one launch of 32: launches of 32 + 4, 3 x 12 and 36 x 1."""
    m, scans, poses, inv = _seam_and_rows_scene(np.random.default_rng(15), 36, 2.5, nonrigid=(33,))
    _check(m, scans, poses, inv, 2.5)


def _surface(rng, centre, u, v, half, step):
    a = np.arange(-half[0], half[0] + 1e-9, step)
    b = np.arange(-half[1], half[1] + 1e-9, step)
    A, Bm = np.meshgrid(a, b)
    p = centre + A.reshape(-1, 1) * u + Bm.reshape(-1, 1) * v
    return p + rng.normal(0, step * 0.1, p.shape)


@pytest.mark.parametrize("alpha", [2.5, 1.5])
def test_tiles_at_the_border_the_seam_and_an_occluder_edge(alpha):
    """Dense surfaces in voxel order, so that 128-point tiles are compact and culling decides per tile: a wall across the seam, a ceiling
    and a floor patch at the top / bottom rows, and a background wall behind an occluding board with a gap.  The map is the scene itself
    (static, culled), copies pulled towards the sensor (candidates) and pushed away (occluded)."""
    rng = np.random.default_rng(21)
    ex, ey, ez = np.eye(3)
    parts = [
        _surface(rng, np.array([-12.0, 0.0, 0.0]), ey, ez, (6.0, 3.0), 0.08),                 # wall across the seam (behind the sensor)
        _surface(rng, np.array([4.0, 3.0, 6.0]), ex, ey, (4.0, 4.0), 0.08),                   # ceiling patch: rows beyond the top edge
        _surface(rng, np.array([3.0, -4.0, -5.0]), ex, ey, (4.0, 4.0), 0.08),                 # floor patch: rows beyond the bottom edge
        _surface(rng, np.array([20.0, 0.0, 0.0]), ey, ez, (10.0, 4.0), 0.08),                 # background wall
        _surface(rng, np.array([10.0, -2.0, 0.0]), ey, ez, (2.0, 3.0), 0.06),                 # occluder, left of the gap
        _surface(rng, np.array([10.0, 3.5, 0.0]), ey, ez, (1.5, 3.0), 0.06),                  # occluder, right of the gap
    ]
    scene = np.concatenate(parts)
    K = 6
    poses = np.stack([_pose(0, [0.05 * k, 0.03 * k, 0.0]) for k in range(K)])
    inv = oracle.inverse_poses(poses)
    scans = []
    for k in range(K):
        local = scene - poses[k][:3, 3]
        rows, cols = oracle.reset_rimg_size(alpha)
        r, c, rng_ = oracle.pixel_index(local, rows, cols)
        keep = np.zeros(len(local), bool)                     # the nearest surface point per pixel is what the sensor returns
        order = np.lexsort((rng_, r * cols + c))
        first = np.ones(len(order), bool); first[1:] = (r * cols + c)[order][1:] != (r * cols + c)[order][:-1]
        keep[order[first]] = True
        scans.append(_xyzi(local[keep], 0.0))
    pulled = poses[0][:3, 3] + (scene - poses[0][:3, 3]) * rng.uniform(0.9, 0.99, (len(scene), 1))
    pushed = poses[0][:3, 3] + (scene - poses[0][:3, 3]) * rng.uniform(1.01, 1.3, (len(scene), 1))
    m = oracle.voxel(_xyzi(np.concatenate([scene, pushed, pulled[::7]])), 0.03)
    _check(m, scans, poses, inv, alpha, culled_min=0.001)


def test_steep_pairs_stay_on_the_fast_path():
    """Map points far above and below the field of view round to the outermost guard rows.  Away from the seam and with their row far
    from a rounding boundary (alpha 2.5: rows -3.91 and 128.91), they must be settled by the fast path: a guard row too few would send
    them to the full exact path, which gives the same flags but loses the point of the padding."""
    rng = np.random.default_rng(31)
    n = 20000
    az = rng.uniform(-3.0, 3.0, n)
    el = np.deg2rad(rng.choice([1, -1], n) * rng.uniform(35.0, 80.0, n))
    scan = _xyzi(_sph(az, el, rng.uniform(5.0, 50.0, n)), 0.0)
    m = _xyzi(_sph(az, el, rng.uniform(2.0, 60.0, n)).astype(np.float32))
    I4 = np.eye(4)[None]
    exp = oracle.remove_pass(m, scan, [0, n], I4, oracle.MODE_HD, 2.5)
    with ltr.Context(cull=False) as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(scan, [0, n]); ps = ctx.poses_upload(I4, I4)
        ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)
        assert np.array_equal(ctx.flags_download(mh), exp)
        st = ctx.last_pass_stats()
    assert st[5] <= 1e-2 * st[0], st      # pairs through the full exact path (0.15 % here: columns near a rounding boundary)


@pytest.mark.parametrize("alpha", [2.5, 1.5])
def test_one_background_pixel_inside_a_tile_rectangle(alpha):
    """A wall 5 m from the sensor fills every pixel except one "hole" per 128-point tile of the first half, through which the scan sees
    60 m.  Each tile is a ball of points 15-30 m away (behind the wall); its hole is the pixel of one of its points, so that point is a
    candidate and the tile must not be culled.  Tiles of the second half have no hole of their own; those whose rectangle holds no other
    tile's hole are culled.  Tiles of 1-12 px radius use every window size of the culling's sliding-window maxima, and a hole anywhere
    in the rectangle -- not only where an aligned block or a shorter window would cover it -- must keep the tile."""
    rng = np.random.default_rng(41)
    rows, cols = oracle.reset_rimg_size(alpha)
    ppr = cols / (2 * np.pi)
    n_tiles = 2000                                                          # 256 k points: more than one per pixel, so culling is on
    az0 = rng.uniform(-2.9, 2.9, n_tiles); el0 = np.deg2rad(rng.uniform(-20, 20, n_tiles)); r0 = rng.uniform(15.0, 30.0, n_tiles)
    rad = rng.uniform(1.0, 12.0, n_tiles) / ppr * r0                        # ball radius: 1-12 px at the tile's range
    d = rng.normal(size=(n_tiles, 128, 3)); d /= np.linalg.norm(d, axis=2, keepdims=True)
    pts = _sph(az0, el0, r0)[:, None, :] + d * (rad[:, None, None] * rng.uniform(0, 1, (n_tiles, 128, 1)) ** (1 / 3))
    m = _xyzi(pts.reshape(-1, 3).astype(np.float32))
    r_m, c_m, _ = oracle.pixel_index(m[:, :3], rows, cols)
    holes = set()
    for t in range(n_tiles // 2):
        j = t * 128 + int(rng.integers(128))
        holes.add((int(r_m[j]), int(c_m[j])))
    # one scan return per pixel, at the pixel's centre direction
    rr, cc = np.meshgrid(np.arange(rows), np.arange(1, cols), indexing="ij")
    el = np.deg2rad((1.0 - rr.ravel() / rows) * 50.0 - 25.0)
    az = np.deg2rad(cc.ravel() / cols * 360.0 - 180.0)
    wall = _sph(az, el, np.full(az.shape, 5.0)).astype(np.float32)
    r_s, c_s, _ = oracle.pixel_index(wall, rows, cols)
    hole = np.array([(int(a), int(b)) in holes for a, b in zip(r_s, c_s)])
    scan = _sph(az, el, np.where(hole, 60.0, 5.0)).astype(np.float32)
    I4 = np.eye(4)[None]
    exp = _check(m, [_xyzi(scan, 0.0)], I4, I4, alpha, batches=(1,), culled_min=0.001)
    assert exp[0].sum() >= n_tiles // 4
