"""ltr_remove_pass keeps the scan-side images of a pass (scan range image, test image, sliding-window maxima) and serves them to later passes
on the same scan set, poses, keyframe range and image shape.  Every pass must still flag exactly what the oracle flags and what the same
pass flags with the kept images turned off (LTR_SCAN_IMAGE_CACHE_MB=0): HD, ND and PD passes repeated on one scan set at the remove, revert
and visible-point resolutions, with and without the empty-scan shortcut, on guard-padded (360 degree) and plain (180 degree) images, over
keyframe sub-ranges and at launch batches of 1, 3, 32 and 36.  A set must never be served after its scan set or poses were freed -- also
when the new object gets the freed handle -- or after ltr_scan_images_release; a budget too small for a set falls back to per-launch
images; the sets' storage is reused, not reallocated, from pass to pass; and releasing it gives all its memory back."""
import numpy as np
import pytest

import oracle
import synth
import lt_mapper_b200 as ltr

pytestmark = pytest.mark.gpu

K = 36
ENV = "LTR_SCAN_IMAGE_CACHE_MB"
MODES = ((ltr.MODE_HD, oracle.MODE_HD), (ltr.MODE_ND, oracle.MODE_ND), (ltr.MODE_PD, oracle.MODE_PD))


def _world(sess):
    return np.concatenate([oracle.transform(sess.scan(k), sess.poses[k]) for k in range(sess.K)])


@pytest.fixture(scope="module")
def scene():
    """Scans and poses of the central session; the map is the voxelised query session (another pass through the scene: its moving objects
    are elsewhere, so HD / PD flag points and ND finds map points in front of the scans).  `far` adds one map point 9 km away, which turns
    the empty-scan shortcut off."""
    c, q = synth.make_pair(K, beams=32, az_steps=900)
    inv = np.stack([np.linalg.inv(p) for p in c.poses])
    m = oracle.voxel(_world(q), 0.05)
    far = np.concatenate([m, np.array([[9000.0, 0.0, 0.0, 1.0]], np.float32)])
    other = synth.make_session(0, K, seed=7, beams=32, az_steps=900)   # another scan set of the same keyframe count
    return dict(c=c, inv=inv, m=m, far=far, other=other)


def _expect(m, sess, inv, mode, alpha, hfov, k0=0, k1=None):
    k1 = sess.K if k1 is None else k1
    off = sess.offsets[k0:k1 + 1] - sess.offsets[k0]
    return oracle.remove_pass(m, sess.xyzi[sess.offsets[k0]:sess.offsets[k1]], off, inv[k0:k1], mode, alpha, hfov=hfov)


def _run(ctx, mh, ss, ps, mode, alpha, k0=0, k1=K):
    ctx.remove_pass(mh, ss, ps, mode, alpha, kf_begin=k0, kf_end=k1)
    return ctx.flags_download(mh)


@pytest.mark.parametrize("hfov", [360.0, 180.0])
@pytest.mark.parametrize("alpha", [2.5, float(np.float32(0.95 * 2.5)), 3.0])
@pytest.mark.parametrize("far", [False, True])
def test_repeated_passes_match_oracle_and_uncached(scene, monkeypatch, alpha, hfov, far):
    c, inv = scene["c"], scene["inv"]
    m = scene["far"] if far else scene["m"]
    exp = {lm: _expect(m, c, inv, om, alpha, hfov) for lm, om in MODES}
    assert exp[ltr.MODE_HD].sum() > 0 and exp[ltr.MODE_ND].sum() > 0
    order = [ltr.MODE_HD, ltr.MODE_PD, ltr.MODE_ND, ltr.MODE_HD, ltr.MODE_ND, ltr.MODE_PD, ltr.MODE_HD]
    got = {}
    for cached in (True, False):
        monkeypatch.setenv(ENV, "" if cached else "0")
        with ltr.Context(hfov=hfov) as ctx:
            mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
            launches = []
            for i, mode in enumerate(order):
                l0 = ctx.kernel_launches()
                f = _run(ctx, mh, ss, ps, mode, alpha)
                launches.append(ctx.kernel_launches() - l0)
                assert np.array_equal(f, exp[mode]), (cached, i, mode, np.flatnonzero(f != exp[mode])[:10])
                got[cached, i] = f
            got[cached, "launches"] = launches
    # every pass after the first finds its images: fewer launches than the same pass without kept images
    assert all(a < b for a, b in zip(got[True, "launches"][1:], got[False, "launches"][1:])), (got[True, "launches"], got[False, "launches"])
    for i in range(len(order)):
        assert np.array_equal(got[True, i], got[False, i])


@pytest.mark.parametrize("batch", [1, 3, 32, 36])
def test_subranges_and_batches(scene, batch):
    """Sharded ranks call the pass on their own keyframe blocks; each block gets its own set, and a block's launches read their images at
    the right offset inside it."""
    c, inv, m = scene["c"], scene["inv"], scene["m"]
    ranges = [(0, K), (5, 20), (20, K), (0, 1), (5, 20)]
    with ltr.Context(keyframe_batch=batch) as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        for lm, om in MODES:
            for k0, k1 in ranges:
                f = _run(ctx, mh, ss, ps, lm, 2.5, k0, k1)
                e = _expect(m, c, inv, om, 2.5, 360.0, k0, k1)
                assert np.array_equal(f, e), (batch, lm, k0, k1, np.flatnonzero(f != e)[:10])


def test_freed_scanset_handle_reuse_is_not_served(scene):
    c, other, inv, m = scene["c"], scene["other"], scene["inv"], scene["m"]
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(m); ps = ctx.poses_upload(c.poses, inv)
        ss = ctx.scanset_upload(c.xyzi, c.offsets)
        assert np.array_equal(_run(ctx, mh, ss, ps, ltr.MODE_HD, 2.5), _expect(m, c, inv, oracle.MODE_HD, 2.5, 360.0))
        ctx.scanset_free(ss)
        ss2 = ctx.scanset_upload(other.xyzi, other.offsets)
        assert ss2 == ss, "the new scan set must take the freed handle for this test to mean anything"
        e = _expect(m, other, inv, oracle.MODE_HD, 2.5, 360.0)
        assert not np.array_equal(e, _expect(m, c, inv, oracle.MODE_HD, 2.5, 360.0))
        assert np.array_equal(_run(ctx, mh, ss2, ps, ltr.MODE_HD, 2.5), e)


def test_freed_poses_handle_reuse_is_not_served(scene):
    """New poses behind the same handle: the images do not depend on the poses, but the shortcut of the test image does (how far the map
    lies from the keyframe origins), so the set is keyed on the poses as well.  Here the new poses move every keyframe 8 km away."""
    c, inv, m = scene["c"], scene["inv"], scene["m"]
    moved = c.poses.copy()
    moved[:, 0, 3] += 8000.0
    inv_m = np.stack([np.linalg.inv(p) for p in moved])
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets)
        ps = ctx.poses_upload(c.poses, inv)
        for lm, om in MODES:
            assert np.array_equal(_run(ctx, mh, ss, ps, lm, 2.5), _expect(m, c, inv, om, 2.5, 360.0))
        ctx.poses_free(ps)
        ps2 = ctx.poses_upload(moved, inv_m)
        assert ps2 == ps
        for lm, om in MODES:
            assert np.array_equal(_run(ctx, mh, ss, ps2, lm, 2.5), _expect(m, c, inv_m, om, 2.5, 360.0)), lm


def test_release_rebuilds_and_returns_memory(scene):
    c, inv, m = scene["c"], scene["inv"], scene["m"]
    with ltr.Context() as ctx:
        mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
        e = _expect(m, c, inv, oracle.MODE_HD, 2.5, 360.0)
        l0 = ctx.kernel_launches(); assert np.array_equal(_run(ctx, mh, ss, ps, ltr.MODE_HD, 2.5), e); first = ctx.kernel_launches() - l0
        live_held = ctx.memory_stats()[0]
        ctx.scan_images_release(free_storage=True)
        live_base = ctx.memory_stats()[0]
        assert live_base < live_held
        l0 = ctx.kernel_launches(); assert np.array_equal(_run(ctx, mh, ss, ps, ltr.MODE_HD, 2.5), e)
        assert ctx.kernel_launches() - l0 == first, "after a release the pass builds its images again"
        l0 = ctx.kernel_launches(); assert np.array_equal(_run(ctx, mh, ss, ps, ltr.MODE_HD, 2.5), e)
        assert ctx.kernel_launches() - l0 < first
        # dropping the sets keeps their storage: the next pass rebuilds its images in it without allocating
        ctx.scan_images_release(free_storage=False)
        assert ctx.memory_stats()[0] == live_held
        l0 = ctx.kernel_launches(); assert np.array_equal(_run(ctx, mh, ss, ps, ltr.MODE_HD, 2.5), e)
        assert ctx.kernel_launches() - l0 == first
        assert ctx.memory_stats()[0] == live_held
        # two resolutions held at once, then smaller ones reuse the two blocks, and a release gives every byte back
        for a in (2.5, 2.375, 2.0, 1.9, 2.5):
            assert np.array_equal(_run(ctx, mh, ss, ps, ltr.MODE_HD, a), _expect(m, c, inv, oracle.MODE_HD, a, 360.0)), a
        held2 = ctx.memory_stats()[0]
        for a in (2.0, 1.9, 1.5, 2.5, 2.375):
            _run(ctx, mh, ss, ps, ltr.MODE_HD, a)
            assert ctx.memory_stats()[0] == held2, "the storage only grows past its largest set"
        ctx.scan_images_release(free_storage=True)
        assert ctx.memory_stats()[0] == live_base
        # freeing the scan set drops its sets: the same pass on a new upload rebuilds them
        _run(ctx, mh, ss, ps, ltr.MODE_HD, 2.5)
        ctx.scanset_free(ss)
        ss = ctx.scanset_upload(c.xyzi, c.offsets)
        l0 = ctx.kernel_launches(); assert np.array_equal(_run(ctx, mh, ss, ps, ltr.MODE_HD, 2.5), e)
        assert ctx.kernel_launches() - l0 == first


def test_over_budget_falls_back_to_per_launch_images(scene, monkeypatch):
    c, inv, m = scene["c"], scene["inv"], scene["m"]
    counts = {}
    for setting in ("0", "1"):   # off, and a 1 MiB budget no set fits
        monkeypatch.setenv(ENV, setting)
        with ltr.Context() as ctx:
            mh = ctx.cloud_upload(m); ss = ctx.scanset_upload(c.xyzi, c.offsets); ps = ctx.poses_upload(c.poses, inv)
            live0 = None
            n = []
            for lm, om in MODES + MODES:
                l0 = ctx.kernel_launches()
                assert np.array_equal(_run(ctx, mh, ss, ps, lm, 2.5), _expect(m, c, inv, om, 2.5, 360.0)), (setting, lm)
                n.append(ctx.kernel_launches() - l0)
                if live0 is None:
                    live0 = ctx.memory_stats()[0]
                assert ctx.memory_stats()[0] == live0, "nothing may be kept"
            counts[setting] = n
    assert counts["0"] == counts["1"]
