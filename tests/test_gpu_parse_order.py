"""Visible-point extraction (ltr_parse_projected) with the near-to-far tile order of the deferred true-minimum mode: the output
must be bit-identical for fast_path 0 (reference arithmetic only), 1 and 2 (fast path, tiles claimed near to far), and equal to
the oracle, on maps with pile-ups in the clamped rows, occluded patches, equal ranges, pixel-boundary points and non-Morton order."""
import numpy as np
import pytest

import oracle
import synth
import lt_mapper_b200 as ltr

pytestmark = pytest.mark.gpu

ALPHA = 3.0


def _cloud(xyz, intensity=0.0):
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    return np.concatenate([xyz, np.full((len(xyz), 1), intensity, np.float32)], 1)


def _sphere_dirs(az_deg, el_deg):
    az, el = np.radians(az_deg), np.radians(el_deg)
    return np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], -1)


def _run(m, c, inv, batch, kfs):
    """Visible points of keyframes [0, K) for fast_path 0 / 1 / 2, compared bit for bit with each other and, for the keyframes kfs,
    with the oracle; returns the fast path's `best` atomics per pair."""
    out, atomics = [], 0.0
    for fast, cull in ((False, False), (True, False), (True, True)):
        with ltr.Context(fast_path=fast, cull=cull, keyframe_batch=batch) as ctx:
            mh = ctx.cloud_upload(m)
            ps = ctx.poses_upload(c.poses, inv)
            vis = ctx.parse_projected(mh, ps, 0, c.K, ALPHA)
            st = ctx.last_pass_stats()
            out.append(ctx.scanset_download(vis))
            if fast:
                assert st[6] == 0            # nothing is culled in the true-minimum mode
                atomics = st[3] / max(st[0], 1.0)
    for pts, off in out[1:]:
        assert np.array_equal(off, out[0][1])
        assert np.array_equal(pts.view(np.uint32), out[0][0].view(np.uint32))
    pts, off = out[2]
    for k in kfs:
        e, _ = oracle.parse_projected(m, inv[k], ALPHA)
        assert np.array_equal(pts[off[k]:off[k + 1]].view(np.uint32), e.view(np.uint32)), k
    return atomics


def _adversarial(rng, c, inv):
    """The real map in voxel (Morton) order plus structures placed around keyframe 0's sensor origin."""
    merged = np.concatenate([oracle.transform(c.scan(k), c.poses[k]) for k in range(c.K)])
    base = oracle.voxel(merged, 0.1)
    o = c.poses[0][:3, 3]
    parts = {}
    # pile-ups in the clamped rows: wall tops far above +25 deg fall into row 0, ground within ~4 m below the sensor into the last row
    d = _sphere_dirs(rng.uniform(0, 360, 20000), rng.uniform(30, 80, 20000))
    parts["pile_top"] = o + d * rng.uniform(5, 40, (20000, 1))
    d = _sphere_dirs(rng.uniform(0, 360, 20000), rng.uniform(-85, -30, 20000))
    parts["pile_bottom"] = o + d * rng.uniform(0.5, 4, (20000, 1))
    # an occluder (dense plate at 8 m) in front of a dense patch at 30 m, both inside a 20 x 10 deg window
    d = _sphere_dirs(rng.uniform(40, 60, 40000), rng.uniform(-5, 5, 40000))
    parts["patch"] = o + d * rng.uniform(30.0, 30.5, (40000, 1))
    parts["occluder"] = o + d[:20000] * 8.0
    # equal ranges: exact duplicates (index ties) and points on one sphere of radius 25 m
    dup = base[rng.integers(len(base), size=5000)]
    dups = np.concatenate([dup, dup, dup])     # appended after the voxelisation below, which would merge them
    parts["shell"] = o + _sphere_dirs(rng.uniform(100, 140, 20000), rng.uniform(-20, 20, 20000)) * 25.0
    # points straddling pixel boundaries: azimuth / elevation on the pixel edges of keyframe 0's image (1 / 3 deg per pixel at alpha 3)
    rows, cols = ltr.reset_rimg_size(ALPHA)
    ca = (np.arange(200, 260) / cols) * 360.0 - 180.0
    ra = 25.0 - (np.arange(60, 90) / rows) * 50.0
    A, E = np.meshgrid(ca, ra)
    edge = _sphere_dirs(A.ravel(), E.ravel())
    parts["edges"] = np.concatenate([o + edge * r for r in (12.0, 12.0 + 1e-5, 40.0)])
    extra = oracle.voxel(_cloud(np.concatenate(list(parts.values())), 1.0), 0.01)
    return np.concatenate([base, extra, dups])


@pytest.mark.parametrize("batch", [3, 32])
def test_near_to_far_order_matches_exact_and_oracle(batch):
    rng = np.random.default_rng(7)
    c = synth.make_pair(34, beams=16, az_steps=600)[0]
    inv = oracle.inverse_poses(c.poses)
    m = _adversarial(rng, c, inv)
    atomics = _run(m, c, inv, batch, (0, 1, 17, c.K - 1))
    print(f"batch {batch}: N={len(m)} best atomics per pair {atomics:.4f}")
    assert atomics > 0


def test_near_to_far_order_real_map(small_pair, small_maps):
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)
    _run(small_maps[0], c, inv, 3, range(c.K))


def test_shuffled_map(small_pair, small_maps):
    """Shuffled (non-Morton) order: every tile spans the scene, so the tile distances say little; the result must not change."""
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)
    m = small_maps[0][np.random.default_rng(3).permutation(len(small_maps[0]))]
    _run(m, c, inv, 3, (0, c.K - 1))
