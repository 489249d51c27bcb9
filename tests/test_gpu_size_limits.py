"""The map projection and the load-time voxel grid at their size limits, bit for bit against the oracle and the host restatement.

A. The fast map projection holds a pixel in 18 bits of its queue entry (q_pack, project_fast.cuh), so plan_pass sends an image of more than
   2^18 pixels to the exact kernel even with the fast path on.  Images of 259 920 pixels (guard-padded, whose padded test image is past
   2^18), of exactly 2^18 pixels (general elevation path at 90 x 360, whose last pixel is 0x3ffff; clamped columns at 64 x 256), of 260 100
   pixels at 10 x 360 (184 guard rows, a padded image of 1.39 M pixels) and of 262 625 pixels, just past the limit.  Synthetic scans plus
   rays onto the first and last rows and columns, the corners and the guard rows, with map points in front of and behind each return;
   HD, ND and PD flags, visible points and a scan range image at keyframe batches 1 and 32 over 35 keyframes.
B. The exact path runs launches of up to 400 keyframes (12 doubles of shared memory each): 437 keyframes in launches of 400 + 37.
C. A kept scan-image set is built in launches of at most 1 024 keyframes (build_scan_images): passes over 1 100 keyframes with the sets on
   and off.
D. The voxel grid runs in launches of at most 64 Mi points (voxel_grid_run), its scratch indexed from each launch's first scan:
   LTR_VOXEL_GRID_CHUNK_POINTS splits small inputs into many launches, and 70 M points take two launches at the real limit.

The tests without the gpu mark check on the CPU, with host restatements of plan_pass, make_fast_cfg and the launch splits, that every
input takes the path its GPU test claims.
"""
import math

import numpy as np
import pytest

import oracle
import synth
import lt_mapper_b200 as ltr
from lt_mapper_b200 import removert
from test_gpu_voxel_grid import voxel_points

F32 = np.float32
MODES = ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_ND, oracle.MODE_ND), (ltr.MODE_PD, oracle.MODE_PD))
FAST_PIXEL_LIMIT = 1 << 18      # plan_pass: the pixel field of the fast path's queue entry
FAST_MAX_BATCH = 32             # kFastMaxBatch
EXACT_MAX_BATCH = 400           # plan_pass: keyframes per launch of map_project_kernel
IMAGE_CHUNK = 1024              # kImageChunk
PYR_LEVELS = 5                  # kPyrLevels
VG_CHUNK_POINTS = 64 << 20      # kVgChunkPoints
EL_POLY_ERR = 0.9e-7            # kElPolyErr
VG_KNOB = "LTR_VOXEL_GRID_CHUNK_POINTS"
CACHE_KNOB = "LTR_SCAN_IMAGE_CACHE_MB"
CACHE_MB = "8192"               # fixed: the default budget, a quarter of the free memory of a shared device, could turn the sets off


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def same(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


# ---------------------------------------------------------------------------------------------------------------- host restatements
def fast_cfg(rows, cols, vfov, hfov):
    """make_fast_cfg's el_direct, pad_ok, pad_g and pad_npx."""
    ppr_r = rows * 180.0 / (math.pi * vfov)
    el_direct = (math.atan(0.5) - 0.5 * vfov * math.pi / 180.0) * ppr_r >= 1.0
    el_max = math.atan(0.5) + EL_POLY_ERR
    r_top = math.floor(0.5 * rows - el_max * ppr_r - 1.0e-3 + 0.5)
    r_bot = math.floor(0.5 * rows + el_max * ppr_r + 1.0e-3 + 0.5)
    pad_ok = el_direct and hfov == 360.0
    pad_g = max(-r_top, r_bot - (rows - 1), 0) if pad_ok else 0
    return dict(el_direct=el_direct, pad_ok=pad_ok, pad_g=pad_g, pad_npx=(rows + 2 * pad_g) * (cols + 1))


def plan(vfov, hfov, alpha, fast, batch, nkf):
    """plan_pass: (rows, cols, fast path taken, keyframes per launch)."""
    rows, cols = oracle.reset_rimg_size(alpha, vfov, hfov)
    use_fast = fast and rows * cols <= FAST_PIXEL_LIMIT
    return rows, cols, use_fast, max(1, min(batch, FAST_MAX_BATCH if use_fast else EXACT_MAX_BATCH, nkf))


def image_chunks(k0, k1):
    """build_scan_images: the keyframe ranges of its launches over [k0, k1)."""
    return [(k0 + c0, k0 + min(c0 + IMAGE_CHUNK, k1 - k0)) for c0 in range(0, k1 - k0, IMAGE_CHUNK)]


def vg_launches(off, chunk):
    """voxel_grid_run: (scratch points, [(k0, k1) of each launch])."""
    off = [int(v) for v in off]
    K = len(off) - 1
    max_chunk = max(max(off[k + 1] - off[k] for k in range(K)), min(off[K], chunk))
    out, k0 = [], 0
    while k0 < K:
        k1 = k0 + 1
        while k1 < K and off[k1 + 1] - off[k0] <= max_chunk:
            k1 += 1
        out.append((k0, k1))
        k0 = k1
    return max_chunk, out


# ---------------------------------------------------------------------------------------------------------------- A: the pixel limit
# name: (vfov, hfov, alpha, rows, cols, fast path with fast_path on, guard-padded test image, pad_g, padded pixels)
SHAPES = {
    "50x360_a3.8": (50.0, 360.0, 3.8, 190, 1368, True, True, 7, 279_276),
    "50x360_a3.82": (50.0, 360.0, 3.82, 191, 1375, False, True, 7, 282_080),
    "90x360_2^18": (90.0, 360.0, float(F32(1024 / 360)), 256, 1024, True, False, 0, 262_400),
    "64x256_2^18": (64.0, 256.0, 4.0, 256, 1024, True, False, 0, 262_400),
    "10x360_a8.5": (10.0, 360.0, 8.5, 85, 3060, True, True, 184, 1_386_633),
}
K_EDGE = 35         # one launch of 32 and a remainder of 3


def _sph(az, el, r):
    ce = np.cos(el)
    return np.stack([r * ce * np.cos(az), r * ce * np.sin(az), r * np.sin(el)], 1)


def _xyzi(p, i=1.0):
    return np.concatenate([np.asarray(p, F32).reshape(-1, 3), np.full((len(p), 1), i, F32)], 1)


def _world(sess):
    return np.concatenate([oracle.transform(sess.scan(k), sess.poses[k]) for k in range(sess.K)])


def edge_rays(vfov, hfov, rows, cols, rng):
    """(az, el) [rad] onto the extreme pixels: the first and last rows (inside them, just past the edge of the field of view and far past
    it, where the row clamps) at random azimuths; column 0 and the last column (the last one outside the seam band: az = pi - 0.75 px;
    beyond the edge, where the column clamps, for fields of view under 360 degrees) at random elevations; every corner; elevations
    between the edge of the field of view and past atan(0.5) (the guard rows of a padded test image); and random rays inside."""
    row, col = np.deg2rad(vfov / rows), np.deg2rad(hfov / cols)
    hv, hh = np.deg2rad(vfov / 2), np.deg2rad(hfov / 2)
    top = np.array([hv - 0.25 * row, hv + 0.3 * row, min(hv + np.deg2rad(20.0), np.deg2rad(85.0))])
    els = np.concatenate([top, -top])
    az_edge = [hh - 0.75 * col, -hh + 0.25 * col] + ([hh + np.deg2rad(5.0), -hh - np.deg2rad(5.0)] if hfov < 360.0 else [])
    az_edge = np.array(az_edge)
    rnd_az = lambda n: rng.uniform(-0.95 * hh, 0.95 * hh, n)
    rnd_el = lambda n: rng.uniform(-0.95 * hv, 0.95 * hv, n)
    g_hi = max(hv, math.atan(0.5)) + np.deg2rad(2.0)
    guard = rng.choice([1.0, -1.0], 60) * rng.uniform(hv, g_hi, 60)
    az = np.concatenate([rnd_az(20 * len(els)), np.repeat(az_edge, 20), np.repeat(az_edge, len(els)), rnd_az(60), rnd_az(100)])
    el = np.concatenate([np.repeat(els, 20), rnd_el(20 * len(az_edge)), np.tile(els, len(az_edge)), guard, rnd_el(100)])
    return az, el


@pytest.fixture(scope="module")
def edge_base():
    """Scans and poses of one synthetic session; the map is the other session, voxelised (more points than any image has pixels)."""
    c, q = synth.make_pair(K_EDGE, beams=32, az_steps=900)
    return c, oracle.voxel(_world(q), 0.1)


def edge_scene(base, shape):
    """(map, scans, offsets, poses, inverse poses, first edge map point): the synthetic scans plus, per keyframe, a return on every edge
    ray and map points in front of it, just behind it and far behind it."""
    c, m = base
    vfov, hfov, _, rows, cols = SHAPES[shape][:5]
    rng = np.random.default_rng(100 + list(SHAPES).index(shape))
    scans, mpts = [], []
    for k in range(c.K):
        az, el = edge_rays(vfov, hfov, rows, cols, rng)
        rs = rng.uniform(3.0, 60.0, len(az))
        scans.append(np.concatenate([c.scan(k), _xyzi(_sph(az, el, rs), 0.0)]))
        for f in (rng.uniform(0.3, 0.95, len(az)), 1.0 + rng.uniform(0.0, 0.004, len(az)), rng.uniform(1.05, 2.0, len(az))):
            mpts.append(oracle.transform(_xyzi(_sph(az, el, rs * f)), c.poses[k]))
    off = np.concatenate([[0], np.cumsum([len(s) for s in scans])]).astype(np.int64)
    inv = np.stack([np.linalg.inv(p) for p in c.poses])
    return np.concatenate([m] + mpts), np.concatenate(scans), off, c.poses, inv, len(m)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
def test_projection_at_the_pixel_limit(edge_base, shape):
    vfov, hfov, alpha, rows, cols, fast = SHAPES[shape][:6]
    m, xyzi, off, poses, inv, n_base = edge_scene(edge_base, shape)
    exp = {lm: oracle.remove_pass(m, xyzi, off, inv, om, alpha, vfov=vfov, hfov=hfov) for lm, om in MODES}
    for lm, e in exp.items():
        assert 0 < e[n_base:].sum() < len(e) - n_base, (lm, "the edge rays must flag some of their map points, not all")
    vis = [oracle.parse_projected(m, inv[k], alpha, vfov=vfov, hfov=hfov)[0] for k in range(K_EDGE)]
    kf = K_EDGE - 1
    rimg = oracle.scan2rimg(xyzi[off[kf]:off[kf + 1]], rows, cols, vfov=vfov, hfov=hfov)
    for B in (1, 32):
        for fast_on, cull in ((False, False), (True, False), (True, True)):
            cfg = (B, fast_on, cull)
            with ltr.Context(vfov=vfov, hfov=hfov, fast_path=fast_on, cull=cull, keyframe_batch=B) as ctx:
                mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(xyzi, off); ps = ctx.poses_upload(poses, inv)
                for lm, _ in MODES:
                    ctx.remove_pass(mh, ss, ps, lm, alpha)
                    got = ctx.flags_download(mh)
                    assert np.array_equal(got, exp[lm]), (cfg, lm, np.flatnonzero(got != exp[lm])[:10])
                    settled_fast = ctx.last_pass_stats()[1]
                    assert (settled_fast > 0) == (fast_on and fast), (cfg, lm, settled_fast)
                h = ctx.parse_projected(mh, ps, 0, K_EDGE, alpha)
                assert (ctx.last_pass_stats()[1] > 0) == (fast_on and fast), cfg
                pts, poff = ctx.scanset_download(h)
                ctx.scanset_free(h)
                for k in range(K_EDGE):
                    assert same(pts[poff[k]:poff[k + 1]], vis[k]), (cfg, k)
                assert same(ctx.debug_scan_rimg(ss, kf, alpha), rimg), cfg


def test_selfcheck_shapes_take_their_paths():
    for name, (vfov, hfov, alpha, rows, cols, fast, padded, pad_g, pad_npx) in SHAPES.items():
        assert oracle.reset_rimg_size(alpha, vfov, hfov) == (rows, cols), name
        r, c, use_fast, B = plan(vfov, hfov, alpha, True, 32, K_EDGE)
        assert use_fast == fast and B == 32, name
        assert plan(vfov, hfov, alpha, False, 32, K_EDGE)[2:] == (False, 32), name
        fc = fast_cfg(rows, cols, vfov, hfov)
        assert (fc["pad_ok"], fc["pad_g"], fc["pad_npx"]) == (padded, pad_g, pad_npx), (name, fc)
        assert fc["el_direct"] == padded, name
        if padded and fast:
            assert pad_npx > FAST_PIXEL_LIMIT, name                        # the padded index is past 2^18; the pixel it is packed as is not
            assert FAST_MAX_BATCH * pad_npx < (1 << 31), name               # keyframe 31's padded image: an int offset in the kernel
    assert K_EDGE > FAST_MAX_BATCH and K_EDGE % FAST_MAX_BATCH                # batch 32: a full launch (k up to 31) and a remainder
    npx = {n: s[3] * s[4] for n, s in SHAPES.items()}
    assert npx["50x360_a3.8"] == 259_920 and npx["50x360_a3.82"] == 262_625 and npx["10x360_a8.5"] == 260_100
    assert npx["90x360_2^18"] == npx["64x256_2^18"] == FAST_PIXEL_LIMIT


@pytest.mark.parametrize("shape", list(SHAPES))
def test_selfcheck_edge_rays_reach_the_extreme_pixels(shape):
    """The rays land on every corner (at 2^18 pixels the last one is pixel 0x3ffff), the whole first and last row and column, the guard
    rows of a padded image, and the last column away from the seam band."""
    vfov, hfov, _, rows, cols, _, padded, pad_g, _ = SHAPES[shape]
    az, el = edge_rays(vfov, hfov, rows, cols, np.random.default_rng(1))
    r, c, _ = oracle.pixel_index(_sph(az, el, np.full(len(az), 20.0)), rows, cols, vfov=vfov, hfov=hfov)
    px = r.astype(np.int64) * cols + c
    for corner in (0, cols - 1, (rows - 1) * cols, rows * cols - 1):
        assert (px == corner).any(), (shape, corner)
    if rows * cols == FAST_PIXEL_LIMIT:
        assert px.max() == 0x3ffff
    assert (r == 0).sum() >= 20 and (r == rows - 1).sum() >= 20 and (c == 0).sum() >= 20 and (c == cols - 1).sum() >= 20
    last = np.isclose(az, np.deg2rad(hfov / 2 - 0.75 * hfov / cols))
    assert last.any() and (c[last] == cols - 1).all()
    assert (np.abs(az[last]) < np.pi - 0.5 * np.deg2rad(hfov / cols)).all()  # outside the seam band of az_seam_lim
    if padded:
        # unclamped row of the reference arithmetic: a ray whose row is above 0 or below rows - 1 by at most pad_g rounds into a guard row
        v = rows * (1.0 - (np.rad2deg(el) + vfov / 2) / vfov)
        guard = ((v < -0.5) & (v >= -pad_g - 0.5)) | ((v >= rows - 0.5) & (v < rows - 0.5 + pad_g))
        assert guard.sum() >= 20, shape


# ---------------------------------------------------------------------------------------------------------------- B: 400-keyframe launches
K_BIG = 437
BIG_CONFIGS = ((False, 400, 2.5), (False, 1000, 2.5), (True, 400, 3.82))   # (fast path, keyframe_batch, alpha)


def big_scene():
    c, q = synth.make_pair(K_BIG, beams=8, az_steps=90)
    return c, oracle.voxel(_world(q), 0.3)


@pytest.fixture(scope="module")
def big_batch():
    c, m = big_scene()
    inv = np.stack([np.linalg.inv(p) for p in c.poses])
    cache = {}

    def expect(alpha):
        if alpha not in cache:
            flags = {lm: oracle.remove_pass(m, c.xyzi, c.offsets, inv, om, alpha) for lm, om in MODES}
            cache[alpha] = flags, [oracle.parse_projected(m, inv[k], alpha)[0] for k in range(K_BIG)]
        return cache[alpha]
    return c, m, inv, expect


@pytest.mark.gpu
@pytest.mark.parametrize("fast,batch,alpha", BIG_CONFIGS)
def test_exact_launches_of_400_keyframes(big_batch, fast, batch, alpha):
    c, m, inv, expect = big_batch
    flags, vis = expect(alpha)
    with ltr.Context(fast_path=fast, keyframe_batch=batch) as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        for lm, _ in MODES:
            ctx.profile_reset()
            ctx.remove_pass(mh, ss, ps, lm, alpha)
            got = ctx.flags_download(mh)
            assert np.array_equal(got, flags[lm]), (lm, np.flatnonzero(got != flags[lm])[:10])
            assert ctx.profile_get()[1] == 2, (lm, "two launches: 400 + 37 keyframes")
            assert ctx.last_pass_stats()[1] == 0, lm
        ctx.profile_reset()
        h = ctx.parse_projected(mh, ps, 0, K_BIG, alpha)
        assert ctx.profile_get()[5] == 2
        pts, poff = ctx.scanset_download(h)
        ctx.scanset_free(h)
        for k in range(K_BIG):
            assert same(pts[poff[k]:poff[k + 1]], vis[k]), k
        if fast:
            # below 2^18 pixels the same setting takes the fast path, in launches of 32
            ctx.profile_reset()
            ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)
            assert np.array_equal(ctx.flags_download(mh), expect(2.5)[0][ltr.MODE_HD])
            assert ctx.profile_get()[1] == math.ceil(K_BIG / FAST_MAX_BATCH) and ctx.last_pass_stats()[1] > 0


def test_selfcheck_exact_launches():
    for fast, batch, alpha in BIG_CONFIGS:
        rows, cols, use_fast, B = plan(50.0, 360.0, alpha, fast, batch, K_BIG)
        assert (use_fast, B) == (False, EXACT_MAX_BATCH) and math.ceil(K_BIG / B) == 2
        assert B * 12 * 8 <= 48 * 1024                                 # the launch's inverse poses in the default shared memory
    assert plan(50.0, 360.0, 2.5, True, 400, K_BIG)[2:] == (True, FAST_MAX_BATCH)
    c, m = big_scene()
    assert c.K == K_BIG and len(m) <= 200_000


# ---------------------------------------------------------------------------------------------------------------- C: kept sets past 1 024 keyframes
K_SET = 1100
SET_RANGES = ((0, K_SET), (3, K_SET), (1020, 1030))
SET_BLOCKS = (0, 3, 1020, 1030, K_SET)     # every range is a union of consecutive blocks; its flags are the union of theirs
SET_ALPHAS = (1.0, 2.5)


def set_scene():
    c, q = synth.make_pair(K_SET, beams=8, az_steps=90)
    return c, oracle.voxel(_world(q), 0.5)


@pytest.fixture(scope="module")
def kept_sets():
    c, m = set_scene()
    return c, m, np.stack([np.linalg.inv(p) for p in c.poses])


@pytest.mark.gpu
@pytest.mark.parametrize("alpha", SET_ALPHAS)
def test_kept_scan_image_sets_past_1024_keyframes(kept_sets, monkeypatch, alpha):
    c, m, inv = kept_sets
    o = c.offsets
    block = {}
    for b0, b1 in zip(SET_BLOCKS[:-1], SET_BLOCKS[1:]):
        for _, om in MODES:
            block[b0, om] = oracle.remove_pass(m, c.xyzi[o[b0]:o[b1]], o[b0:b1 + 1] - o[b0], inv[b0:b1], om, alpha)
    exp = {}
    for k0, k1 in SET_RANGES:
        for _, om in MODES:
            exp[k0, om] = np.bitwise_or.reduce([block[b, om] for b in SET_BLOCKS[:-1] if k0 <= b < k1])
            assert exp[k0, om].sum() > 0, (k0, om)
    launches = {}
    for budget in (CACHE_MB, "0"):
        monkeypatch.setenv(CACHE_KNOB, budget)
        with ltr.Context() as ctx:
            mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, o); ps = ctx.poses_upload(c.poses, inv)
            for k0, k1 in SET_RANGES:
                for lm, om in MODES:
                    for rep in range(2):
                        l0 = ctx.kernel_launches()
                        ctx.remove_pass(mh, ss, ps, lm, alpha, kf_begin=k0, kf_end=k1)
                        launches[budget, k0, lm, rep] = ctx.kernel_launches() - l0
                        got = ctx.flags_download(mh)
                        assert np.array_equal(got, exp[k0, om]), (budget, k0, k1, lm, rep, np.flatnonzero(got != exp[k0, om])[:10])
    for k0, _ in SET_RANGES:
        for lm, _ in MODES:
            assert launches[CACHE_MB, k0, lm, 1] < launches["0", k0, lm, 1], (k0, lm, "the repeated pass must find its images in the set")


def test_selfcheck_kept_sets():
    c, m = set_scene()
    assert c.K == K_SET
    assert [len(image_chunks(k0, k1)) for k0, k1 in SET_RANGES] == [2, 2, 1]
    assert image_chunks(3, K_SET)[1] == (1027, K_SET)
    for alpha in SET_ALPHAS:
        rows, cols, use_fast, B = plan(50.0, 360.0, alpha, True, 32, K_SET)
        npx, pad_npx = rows * cols, fast_cfg(rows, cols, 50.0, 360.0)["pad_npx"]
        assert use_fast and B <= 32 and len(m) >= npx            # tile culling on: the sets hold the window table
        if alpha == 1.0:
            assert (npx, pad_npx) == (18_000, 20_216)
        # storage of the two large sets (rimg | timg | pyr) fits the fixed budget together
        set_bytes = K_SET * 4 * (npx + pad_npx + PYR_LEVELS * npx)
        assert 2 * set_bytes < int(CACHE_MB) << 20, (alpha, set_bytes)


# ---------------------------------------------------------------------------------------------------------------- D: voxel grid launches
KNOB_CHUNKS = (1, 1000, 4096)
KNOB_SIZES = (0, 300, 1500, 0, 120, 900, 640, 0, 250, 800, 700, 410, 990, 0, 333, 870, 512, 64, 2, 0)
KNOB_OVERFLOW = (9, 12, 16, 18)
REAL_SIZES = (14_000_000,) * 5


def knob_scans():
    """Scans of the order-sensitive voxel_points of test_gpu_voxel_grid (voxels of about 4 points, intensities 1e7 and ~1 mixed): empty
    scans first, inside and last, one of 1 500 points -- larger than a chunk of 1 000 -- and overflow-exit scans (one point 3e9 voxels
    out) in the later launches."""
    rng = np.random.default_rng(61)
    parts = []
    for k, n in enumerate(KNOB_SIZES):
        p = voxel_points(rng.integers(0, max(n // 4, 1), n), rng)
        if k in KNOB_OVERFLOW:
            p[1, 0] = F32(3.0e9)
        parts.append(p)
    return np.concatenate(parts), np.concatenate([[0], np.cumsum(KNOB_SIZES)]).astype(np.int64)


def real_size_scans():
    rng = np.random.default_rng(71)
    n = sum(REAL_SIZES)
    x = np.empty((n, 4), F32)
    x[:, :3] = rng.random((n, 3), F32) * F32(100.0)
    x[:, 3] = rng.random(n, F32)
    return x, np.concatenate([[0], np.cumsum(REAL_SIZES)]).astype(np.int64)


def device_voxel_grid(ctx, x, off, leaf):
    h = ctx.scanset_upload(x, off)
    l0 = ctx.kernel_launches()
    o, nov = ctx.voxel_grid_per_keyframe(h, leaf)
    n_launch = ctx.kernel_launches() - l0
    pts, oo = ctx.scanset_download(o)
    ctx.scanset_free(o)
    ctx.scanset_free(h)
    return pts, oo, nov, n_launch


@pytest.mark.gpu
def test_voxel_grid_chunk_knob(monkeypatch):
    x, off = knob_scans()
    exp, exp_off = removert.voxel_grid_scans(x, off, 1.0)
    n_ov = sum(removert.voxel_grid(x[off[k]:off[k + 1]], 1.0)[1] for k in range(len(off) - 1))
    runs = {}
    with ltr.Context() as ctx:
        for chunk in (None,) + KNOB_CHUNKS:
            if chunk is None:
                monkeypatch.delenv(VG_KNOB, raising=False)
            else:
                monkeypatch.setenv(VG_KNOB, str(chunk))
            pts, oo, nov, n_launch = runs[chunk] = device_voxel_grid(ctx, x, off, 1.0)
            assert np.array_equal(oo, exp_off) and same(pts, exp) and nov == n_ov, chunk
    for chunk in KNOB_CHUNKS:
        assert same(runs[chunk][0], runs[None][0]) and np.array_equal(runs[chunk][1], runs[None][1])
        # the other launches of the call are the same: the knob only splits the filter's own launches
        assert runs[chunk][3] - runs[None][3] == len(vg_launches(off, chunk)[1]) - 1, chunk


@pytest.mark.gpu
def test_voxel_grid_of_70m_points_in_two_launches(monkeypatch):
    """Five scans of 14 M points: over 64 Mi points in all, so the filter takes two launches at its real limit (not a knob)."""
    monkeypatch.delenv(VG_KNOB, raising=False)
    x, off = real_size_scans()
    exp, exp_off = removert.voxel_grid_scans(x, off, 0.5)
    with ltr.Context() as ctx:
        one = device_voxel_grid(ctx, x[:1000], [0, 1000], 0.5)[3]    # the launches of a call whose filter takes one launch
        pts, oo, nov, n_launch = device_voxel_grid(ctx, x, off, 0.5)
    assert n_launch == one + 1
    assert nov == 0 and np.array_equal(oo, exp_off) and same(pts, exp)


def test_selfcheck_voxel_grid_launches():
    x, off = knob_scans()
    sizes = np.diff(off)
    assert (sizes == 0).sum() >= 4 and sizes[0] == 0 and sizes[-1] == 0
    ov = [k for k in range(len(sizes)) if sizes[k] and removert.voxel_grid(x[off[k]:off[k + 1]], 1.0)[1]]
    assert ov == list(KNOB_OVERFLOW)
    assert vg_launches(off, VG_CHUNK_POINTS) == (off[-1], [(0, len(sizes))])
    for chunk in KNOB_CHUNKS:
        max_chunk, launches = vg_launches(off, chunk)
        assert max_chunk == max(sizes.max(), chunk) and len(launches) >= 3, chunk
        assert all(off[k1] - off[k0] <= max_chunk for k0, k1 in launches)
        first = launches[0][1]
        assert all(k >= first for k in ov), (chunk, "overflow exits only in later launches")
        assert any(sizes[k0:k1].min() == 0 for k0, k1 in launches[1:]), (chunk, "empty scans in later launches")
    assert vg_launches(off, 1000)[0] == 1500 == sizes.max()           # a scan larger than the chunk sets the scratch
    roff = np.concatenate([[0], np.cumsum(REAL_SIZES)])
    assert roff[-1] > VG_CHUNK_POINTS and vg_launches(roff, VG_CHUNK_POINTS) == (VG_CHUNK_POINTS, [(0, 4), (4, 5)])
