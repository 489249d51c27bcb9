"""Load-time pcl::VoxelGrid on the device (voxel_grid.cu: ltr_voxel_grid, ltr_voxel_grid_per_keyframe, ltrh_load_session_raw and the
cascade promotion) byte for byte against its host restatement (removert.voxel_grid / voxel_grid_scans, io.cpp voxel_grid_span).

Most inputs hold voxels of 3 or more points whose f32 sums depend on the summation order (intensities of about 1e7 and 1 mixed in one
voxel), so an entry order other than libstdc++'s std::sort permutation changes bits; `stable_restatement` proves that for the crafted
inputs by showing that a stable sort of the same entries gives different bits.
"""
import numpy as np
import pytest

import lt_mapper_b200 as ltr
from lt_mapper_b200 import removert
import synth

pytestmark = pytest.mark.gpu

F32 = np.float32


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def same(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


@pytest.fixture(scope="module")
def ctx():
    with ltr.Context(device=0) as c:
        yield c


def device_cloud(ctx, x, leaf):
    h = ctx.cloud_upload(x)
    o, ov = ctx.voxel_grid(h, leaf)
    out = ctx.cloud_download(o).copy()
    ctx.cloud_free(h)
    ctx.cloud_free(o)
    return out, ov


def device_scans(ctx, x, off, leaf):
    h = ctx.scanset_upload(x, off)
    o, nov = ctx.voxel_grid_per_keyframe(h, leaf)
    pts, oo = ctx.scanset_download(o)
    ctx.scanset_free(h)
    ctx.scanset_free(o)
    return pts, oo, nov


def check_cloud(ctx, x, leaf):
    exp, exp_ov = removert.voxel_grid(x, leaf)
    got, ov = device_cloud(ctx, x, leaf)
    assert ov == exp_ov
    assert same(got, exp), f"{len(got)} vs {len(exp)} points"
    return exp, exp_ov


def stable_restatement(x, leaf):
    """voxel_grid_span with a STABLE sort of the entries (finite inputs only): what a wrong permutation would give."""
    x = np.asarray(x, F32)
    inv = F32(1.0) / F32(leaf)
    mn, mx = x[:, :3].min(0), x[:, :3].max(0)
    minb = np.floor(mn * inv).astype(np.int64)
    div = np.floor(mx * inv).astype(np.int64) - minb + 1
    ijk = (np.floor(x[:, :3] * inv) - minb.astype(F32)).astype(np.int64)
    idx = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    order = np.argsort(idx, kind="stable")
    out = []
    i = 0
    while i < len(order):
        j = i
        s = np.zeros(4, F32)
        while j < len(order) and idx[order[j]] == idx[order[i]]:
            s = (s + x[order[j]]).astype(F32)
            j += 1
        out.append(s / F32(j - i))
        i = j
    return np.array(out, F32).reshape(-1, 4)


def voxel_points(keys, rng, per_key=None):
    """Points on the x axis at leaf 1.0: voxel index == key.  Intensities mix 1e7 and ~1 so that sums depend on their order."""
    keys = np.asarray(keys, np.int64)
    n = len(keys)
    x = np.zeros((n, 4), F32)
    x[:, 0] = keys.astype(F32) + F32(0.25) + rng.random(n).astype(F32) * F32(0.5)
    x[:, 1] = rng.random(n).astype(F32) * F32(0.5)
    x[:, 2] = rng.random(n).astype(F32) * F32(0.5)
    big = rng.random(n) < 0.5
    x[:, 3] = np.where(big, rng.choice([F32(1.0e7), F32(-1.0e7)], n), rng.random(n).astype(F32) * F32(3.0) + F32(0.1)).astype(F32)
    return x


def synth_scans(K, seed=7):
    s = synth.make_session(0, K, beams=32, az_steps=900)
    x = s.xyzi.copy()
    off = s.offsets
    rng = np.random.default_rng(seed)
    for k in range(1, K, 2):                       # every other scan shrunk: it never takes the overflow exit
        x[off[k]:off[k + 1], :3] *= F32(0.02)
    x[:, 3] = np.where(rng.random(len(x)) < 0.3, F32(1.0e7), x[:, 3]).astype(F32)
    return x, off


# ------------------------------------------------------------------------------------------------------------------------ scans
@pytest.mark.parametrize("leaf", [0.05, 0.1, 0.3, 1.0])
def test_synth_scans_match_host(ctx, leaf):
    x, off = synth_scans(6)
    exp, exp_off = removert.voxel_grid_scans(x, off, leaf)
    n_ov = sum(removert.voxel_grid(x[off[k]:off[k + 1]], leaf)[1] for k in range(len(off) - 1))
    got, got_off, nov = device_scans(ctx, x, off, leaf)
    assert np.array_equal(got_off, exp_off)
    assert same(got, exp)
    assert nov == n_ov
    if leaf == 0.05:
        assert 0 < n_ov < len(off) - 1, "both exits must be present"


def test_single_voxel_of_1000_points(ctx):
    rng = np.random.default_rng(1)
    x = voxel_points(np.full(1000, 5), rng)
    exp, _ = check_cloud(ctx, x, 1.0)
    assert len(exp) == 1
    assert not same(stable_restatement(x, 1.0), exp), "input does not tell the permutations apart"


@pytest.mark.parametrize("pattern", ["sorted", "reversed", "organ_pipe", "all_equal"])
@pytest.mark.parametrize("n", [600, 5000, 40000])
def test_key_patterns(ctx, pattern, n):
    rng = np.random.default_rng(n)
    u = np.arange(n) // 4                               # every voxel 4 points
    keys = {"sorted": u, "reversed": u[::-1], "organ_pipe": np.concatenate([u[: n // 2], u[: n - n // 2][::-1]]),
            "all_equal": np.zeros(n, np.int64)}[pattern]
    x = voxel_points(keys, rng)
    exp, _ = check_cloud(ctx, x, 1.0)
    assert not same(stable_restatement(x, 1.0), exp), "input does not tell the permutations apart"


@pytest.mark.parametrize("n", [0, 1, 2, 3, 15, 16, 17, 33, 2 ** 17 + 1])
def test_scan_sizes(ctx, n):
    rng = np.random.default_rng(n + 3)
    x = voxel_points(rng.integers(0, max(n // 3, 1), n), rng)
    check_cloud(ctx, x, 1.0)
    if n >= 33:
        assert not same(stable_restatement(x, 1.0), removert.voxel_grid(x, 1.0)[0])


def test_overflow_boundary(ctx):
    """INT32_MAX is a prime, so a product of truncated float extents can equal it only as dx = INT32_MAX -- which no float reaches
    (floats near 2^31 are 128 apart).  The nearest products on either side: 2^31 - 127 (filtered) and 2^31 = INT32_MAX + 1 (exit),
    plus 2047 x 1024 x 1024 (filtered) against 2048 x 1024 x 1024 (exit)."""
    rng = np.random.default_rng(5)
    cases = [((2147483520.0, 0.0, 0.0), False), ((2147483648.0, 0.0, 0.0), True),
             ((2046.5, 1023.5, 1023.5), False), ((2047.5, 1023.5, 1023.5), True)]
    for ext, exp_ov in cases:
        x = voxel_points(rng.integers(0, 40, 300), rng)
        x[:, :3] = (x[:, :3] / F32(40.0)).astype(F32)     # inside [0, 1.1): the box is set by the two corner points
        x[0, :3] = 0.0
        x[1, :3] = np.array(ext, F32)
        _, ov = check_cloud(ctx, x, 1.0)
        assert ov == exp_ov, ext


@pytest.mark.parametrize("where", [0, 1, 7])
@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_non_finite(ctx, where, value, axis):
    """NaN / +-inf in every coordinate, including the first point: std::min/max skip NaN, float -> int conversions of NaN and of
    out-of-range values give 0x80000000..., the int32 index arithmetic wraps."""
    rng = np.random.default_rng(11 + where + axis)
    x = voxel_points(rng.integers(0, 30, 200), rng)
    x[where, axis] = value
    x[where + 20, (axis + 1) % 3] = value
    check_cloud(ctx, x, 1.0)
    check_cloud(ctx, x, 0.05)
    y = x.copy()
    y[:, axis] = value                                     # a whole axis non-finite
    check_cloud(ctx, y, 1.0)


def test_nan_payloads(ctx):
    """x86 NaN results: inf + -inf gives the default NaN 0xffc00000, a NaN operand comes through quieted, and of two NaNs the
    accumulator's wins (CUDA would give 0x7fffffff for all of them)."""
    u = lambda v: np.frombuffer(np.uint32(v).tobytes(), F32)[0]
    x = np.array([[0.5, 0, 0, np.inf], [0.6, 0, 0, -np.inf], [0.7, 0, 0, u(0x7f800001)], [1.5, 0, 0, u(0xffa00005)],
                  [1.6, 0, 0, 2.0], [2.5, 0, 0, u(0x7fc01234)], [2.6, 0, 0, u(0xff800007)]], F32)
    exp, _ = check_cloud(ctx, x, 1.0)
    assert np.isnan(exp[:, 3]).all()


def test_all_nan_scan(ctx):
    x = np.full((40, 4), np.nan, F32)
    check_cloud(ctx, x, 0.5)


@pytest.mark.parametrize("K", [1, 2000])
def test_many_keyframes_mixed_exits(ctx, K):
    rng = np.random.default_rng(K)
    parts, off = [], [0]
    for k in range(K):
        n = int(rng.integers(0, 300)) if k % 7 else 0
        p = voxel_points(rng.integers(0, max(n // 3, 1), n), rng)
        if k % 3 == 1 and n > 1:
            p[1, 0] = F32(3.0e9)                          # extent beyond INT32_MAX voxels: overflow exit
        parts.append(p)
        off.append(off[-1] + n)
    x = np.concatenate(parts) if parts else np.zeros((0, 4), F32)
    off = np.array(off, np.int64)
    exp, exp_off = removert.voxel_grid_scans(x, off, 1.0)
    n_ov = sum(removert.voxel_grid(x[off[k]:off[k + 1]], 1.0)[1] for k in range(K))
    got, got_off, nov = device_scans(ctx, x, off, 1.0)
    assert np.array_equal(got_off, exp_off) and same(got, exp) and nov == n_ov
    if K > 1:
        assert 0 < n_ov < K


@pytest.mark.parametrize("n", [600, 3000])
def test_mcilroy_adversary_reaches_heap_sort(ctx, n):
    """McIlroy's adversary ("A killer adversary for quicksort") against the libstdc++ transcription of test_voxel_grid_sort_model,
    coarsened to voxels of 3 points (it still drives the introsort into its heap-sort branch, whose permutation then decides the sums)."""
    from test_voxel_grid_sort_model import introsort_trace, mcilroy_adversary
    keys = mcilroy_adversary(n) // 3
    assert introsort_trace(keys)["heap_sorts"] > 0
    x = voxel_points(keys, np.random.default_rng(n))
    exp, _ = check_cloud(ctx, x, 1.0)
    assert not same(stable_restatement(x, 1.0), exp), "input does not tell the permutations apart"


def test_invalid_leaf(ctx):
    h = ctx.cloud_upload(np.zeros((4, 4), F32))
    for leaf in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ltr.LtrError):
            ctx.voxel_grid(h, leaf)
    ctx.cloud_free(h)


def test_memory_returns(ctx):
    x, off = synth_scans(4)
    h = ctx.scanset_upload(x, off)
    live0 = ctx.memory_stats()[0]
    o, _ = ctx.voxel_grid_per_keyframe(h, 0.3)
    ctx.scanset_free(o)
    assert ctx.memory_stats()[0] == live0
    ctx.scanset_free(h)


# ------------------------------------------------------------------------------------------------------------------------ orchestrator
def _run_pair(R, c, q):
    R.run_step0()
    R.run_step12()
    R.run_step3()
    out = {}
    for name in ("map_global_curr_", "map_global_updated_", "map_global_updated_strong_"):
        out[name] = R.cloud(name)
    for name in ("keyframe_scans_", "keyframe_scans_updated_", "keyframe_scans_updated_strong_", "keyframe_scans_pd_"):
        out[name] = R.scanset(name)
    return out


def test_load_session_raw_matches_host_filtered_load():
    c, q = synth.make_pair(4, beams=32, az_steps=900)
    leaf = 0.3
    runs = []
    for raw in (True, False):
        with removert.Removerter(device=0, voxel=leaf) as R:
            for sess, s in enumerate((c, q)):
                inv = removert.inverse_poses(s.poses)
                if raw:
                    R.load_session_raw(sess, s.xyzi, s.offsets, s.poses, inv)
                else:
                    x, o = removert.voxel_grid_scans(s.xyzi, s.offsets, leaf)
                    R.load_session(sess, x, o, s.poses, inv)
            runs.append(_run_pair(R, c, q))
    a, b = runs
    for name in a:
        if isinstance(a[name], tuple):
            assert np.array_equal(a[name][1], b[name][1]) and same(a[name][0], b[name][0]), name
        else:
            assert same(a[name], b[name]), name


def test_cascade_promotion_equals_host_filter():
    c, q = synth.make_pair(4, beams=32, az_steps=900)
    leaf = 0.3
    with removert.Removerter(device=0, voxel=leaf) as R:
        for sess, s in enumerate((c, q)):
            R.load_session(sess, s.xyzi, s.offsets, s.poses, removert.inverse_poses(s.poses))
        R.run_step0()
        R.run_step12()
        R.run_step3()
        upd, upd_off = R.scanset("keyframe_scans_updated_")
        exp, exp_off = removert.voxel_grid_scans(upd, upd_off, leaf)
        R.cascade_promote_updated()
        got, got_off = R.scanset("keyframe_scans_")
        assert np.array_equal(got_off, exp_off) and same(got, exp)
