"""Distributed voxeliser (util.cu, ltr_nccl_voxel_centroid_merged) on one GPU, bit for bit against oracle.voxel of the rank-order
concatenation of the local clouds.

ltr_debug_voxel_distributed runs the rank-local stages of the NCCL path for G simulated ranks of one context -- extrema and non-finite
flag, Morton keys and prefix histogram, cuts and the stable grouping by destination, the owner's voxelisation under the global box --
with host reductions and concatenations in place of the collectives, and reports the cuts and the send matrix it decided.  A CPU model of
the prefix histogram, the cut rule and the send matrix checks those, and the tests without the gpu mark use it to show that every scene
takes the path it claims.  The real NCCL path runs at world 1 (NCCL refuses two ranks on one device); world >= 2 over NCCL is
test_gpu_multi.py's.

As in test_gpu_voxel_sort.py the clouds are built so that the f32 sums depend on the order of summation: voxels of 2 to 50 points, about
1e3 m from the origin, intensities of about 1e4 and 1e-3 mixed, shuffled.  Split into contiguous rank blocks, most voxels then have
points on several source ranks, and an owner that loses the source-rank order or the stability of the grouping changes bits.
"""
import ctypes
import functools
from types import SimpleNamespace

import numpy as np
import pytest

import oracle
from test_gpu_voxel_sort import (F32, PAIR_LEAF, SHORTCUT_MIN, bits, boundary_cloud, clustered, define_box, key_bits, morton,
                                 one_per_voxel, pair_cloud)

GS = [1, 2, 3, 4, 5, 8, 16]
HIST_BITS = 12                  # kDistHistBits
UNSUPPORTED, INVALID = -3, -1


# ---------------------------------------------------------------------------------------------------------------- CPU model
def dist_model(locals_, leaf, strict=False):
    """Python restatement of the host decisions of the distributed voxeliser for the local clouds `locals_` (rank order): the global
    box, the prefix bin of every local point, the cuts ub[j] = first bin after the one where the cumulative population reaches
    (j + 1) / G of the total (strict: exceeds it), and send[r, d] = points rank r sends to the owner of range d."""
    G = len(locals_)
    box = define_box(np.concatenate(locals_), leaf)
    depth = box[2]
    hb = min(HIST_BITS, 3 * depth)
    shift = 3 * depth - hb
    nbins = 1 << hb
    bins = [(morton(p, box) >> np.uint64(shift)).astype(np.int64) for p in locals_]
    hist = np.array([np.bincount(b, minlength=nbins) for b in bins], np.int64)
    hg = hist.sum(0)
    total = int(hg.sum())
    cuts, cum = [], 0
    for i in range(nbins):
        if len(cuts) == G - 1:
            break
        cum += int(hg[i])
        while len(cuts) < G - 1 and (cum * G > total * (len(cuts) + 1) if strict else cum * G >= total * (len(cuts) + 1)):
            cuts.append(i + 1)
    cuts += [nbins] * (G - 1 - len(cuts))
    dest = np.searchsorted(np.array(cuts, np.int64), np.arange(nbins), side="right")     # number of cuts ub[j] <= bin
    send = np.array([[int(h[dest == d].sum()) for d in range(G)] for h in hist], np.int64).reshape(G, G)
    return SimpleNamespace(box=box, depth=depth, shift=shift, nbins=nbins, bins=bins, hist=hist, hg=hg, cuts=np.array(cuts, np.uint32),
                           dest=dest, send=send)


def owner_ranges(locals_, m):
    """The cloud each owner receives: its range's points, source rank by source rank, each in local order."""
    G = len(locals_)
    return [np.concatenate([p[m.dest[b] == d] for p, b in zip(locals_, m.bins)]) for d in range(G)]


# ---------------------------------------------------------------------------------------------------------------- scenes
def blocks(p, G):
    """Rank r holds [n r / G, n (r + 1) / G) -- the keyframe blocks of voxeliseMerged and the slices of octreeDownsamplingAppended."""
    n = len(p)
    return [p[n * r // G: n * (r + 1) // G] for r in range(G)]


@functools.lru_cache(None)
def cross_rank_cloud():
    return clustered(40_000, 0.05, 30.0, seed=31)


@functools.lru_cache(None)
def skew_cloud():
    """70 % of the points in clusters inside one prefix bin near the middle of the box, the rest spread over it."""
    spread = clustered(12_000, 0.05, 64.0, seed=41)
    heavy = clustered(28_000, 0.05, 1.5, seed=42, origin=1000.0 + 64.0 * 0.53)
    rng = np.random.default_rng(43)
    p = np.concatenate([spread, heavy])
    return p[rng.permutation(len(p))]


def skew_split(G):
    """The skewed cloud over ranks 0 .. G - 2; the last rank is empty (G >= 2)."""
    p = skew_cloud()
    return blocks(p, 1) if G == 1 else blocks(p, G - 1) + [p[:0]]


@functools.lru_cache(None)
def exact_cut_cloud():
    """Four equal groups of clusters at four corners of the box, in four different first-level octants: the cumulative population is
    exactly 1/4, 2/4 and 3/4 of the total at the last bin of a group, and the bins after it are empty."""
    rng = np.random.default_rng(51)
    parts = [clustered(2000, 0.05, 2.0, seed=52 + c, origin=0.0) + np.array([*o, 0], F32)
             for c, o in enumerate([(1000, 1000, 1000), (1000, 1000, 1030), (1000, 1030, 1000), (1030, 1000, 1000)])]
    p = np.concatenate(parts).astype(F32)
    return p[rng.permutation(len(p))]


# (cloud, leaf, depth) of the octree-depth scenes: depth 1 has 3 code bits (8 bins), depths 2-3 fewer than 12 prefix bits, depth 4 exactly
# 12 (shift 0), depth 6 a shift of 6, depth 17 the pair cloud (its owner ranges take the (key, index) sort), depth 21 the deepest accepted
@functools.lru_cache(None)
def depth_scene(depth):
    if depth == 17:
        return pair_cloud(), PAIR_LEAF
    if depth == 21:
        return boundary_cloud(5000, 1500.0, seed=5), 0.001
    extent = {1: 1.2, 2: 3.0, 3: 6.0, 4: 12.0, 6: 50.0}[depth]
    return clustered(6000, 1.0, extent, seed=60 + depth), 1.0


DEPTHS = [1, 2, 3, 4, 6, 17, 21]


@functools.lru_cache(None)
def shortcut_cloud():
    """A voxelised cloud of about 300k points in octree order: each of two owner ranges holds > 100k points with increasing codes."""
    return one_per_voxel(300_000, 200.0, 0.2, seed=9)


# ---------------------------------------------------------------------------------------------------------------- GPU helpers
@pytest.fixture(scope="module")
def ctx():
    import lt_mapper_b200 as ltr
    c = ltr.Context()
    yield c
    c.close()


def simulate(ctx, locals_, leaf):
    """(voxelised concatenation, cuts, send matrix) of ltr_debug_voxel_distributed over freshly uploaded local clouds."""
    hs = [ctx.cloud_upload(p) for p in locals_]
    try:
        return run_handles(ctx, hs, leaf)
    finally:
        for h in hs:
            ctx.cloud_free(h)


def run_handles(ctx, hs, leaf):
    o, cuts, send = ctx.debug_voxel_distributed(hs, leaf)
    got = ctx.cloud_download(o).copy()
    ctx.cloud_free(o)
    return got, cuts, send


def serial(ctx, p, leaf):
    h = ctx.cloud_upload(p)
    o = ctx.voxel_centroid(h, leaf)
    got = ctx.cloud_download(o).copy()
    ctx.cloud_free(o)
    ctx.cloud_free(h)
    return got


def check(ctx, locals_, leaf, exp=None, got=None):
    """The simulated driver equals oracle.voxel of the concatenation bit for bit, its cuts and send matrix equal the model's, and
    ltr_voxel_centroid of the concatenation gives the same bytes."""
    allp = np.concatenate(locals_)
    if exp is None:
        exp = oracle.voxel(allp, leaf)
    if got is None:
        got = simulate(ctx, locals_, leaf)
    out, cuts, send = got
    m = dist_model(locals_, leaf)
    assert np.array_equal(cuts, m.cuts), (cuts, m.cuts)
    assert np.array_equal(send, m.send), (send, m.send)
    assert out.shape == exp.shape and np.array_equal(bits(out), bits(exp))
    assert np.array_equal(bits(serial(ctx, allp, leaf)), bits(exp))
    return m


def expect_error(ctx, code, fn, launches=None):
    """fn() fails with `code`, returns every byte it took and (launches given) launched exactly that many kernels."""
    import lt_mapper_b200 as ltr
    base, l0 = ctx.memory_stats()[0], ctx.kernel_launches()
    with pytest.raises(ltr.LtrError) as e:
        fn()
    assert e.value.code == code, str(e.value)
    assert ctx.memory_stats()[0] == base
    if launches is not None:
        assert ctx.kernel_launches() - l0 == launches, str(e.value)
    return e.value


# ---------------------------------------------------------------------------------------------------------------- GPU: scenes
def pipeline_locals(ctx, sess, G):
    """Rank r: ltr_merge_scans_global of its keyframe block [K r / G, K (r + 1) / G), as voxeliseMerged gets it."""
    out = []
    for r in range(G):
        k0, k1 = sess.K * r // G, sess.K * (r + 1) // G
        s = sess.subset(k0, k1)
        inv = np.stack([np.linalg.inv(q) for q in s.poses]) if s.K else s.poses
        ss = ctx.scanset_upload(s.xyzi, s.offsets)
        ps = ctx.poses_upload(s.poses, inv)
        m = ctx.merge_scans_global(ss, ps)
        out.append(ctx.cloud_download(m).copy())
        for f, h in ((ctx.cloud_free, m), (ctx.scanset_free, ss), (ctx.poses_free, ps)):
            f(h)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("leaf", [0.05, 0.4])
@pytest.mark.parametrize("G", GS)
def test_pipeline_blocks(ctx, small_pair, G, leaf):
    locals_ = pipeline_locals(ctx, small_pair[0], G)
    if G == 8:
        assert sum(len(p) == 0 for p in locals_) >= 2
    check(ctx, locals_, leaf)


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
def test_appended_slices(ctx, G):
    """Strided views: rank r's cloud is ltr_cloud_slice [n r / G, n (r + 1) / G) of one uploaded cloud (offset = slice start, component
    stride = the parent's capacity), as octreeDownsamplingAppended passes them."""
    p = cross_rank_cloud()[:30_001]
    h = ctx.cloud_upload(p)
    n = len(p)
    views = [ctx.cloud_slice(h, n * r // G, n * (r + 1) // G) for r in range(G)]
    got = run_handles(ctx, views, 0.05)
    for v in views:
        ctx.cloud_free(v)
    assert np.array_equal(bits(ctx.cloud_download(h)), bits(p))      # freeing a view leaves the parent alone
    ctx.cloud_free(h)
    check(ctx, blocks(p, G), 0.05, got=got)


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
def test_cross_rank_voxels(ctx, G):
    check(ctx, blocks(cross_rank_cloud(), G), 0.05, exp=_cross_exp())


@functools.lru_cache(None)
def _cross_exp():
    return oracle.voxel(cross_rank_cloud(), 0.05)


@functools.lru_cache(None)
def _skew_exp():
    return oracle.voxel(skew_cloud(), 0.05)


@functools.lru_cache(None)
def _exact_exp():
    return oracle.voxel(exact_cut_cloud(), 0.05)


@functools.lru_cache(None)
def _depth_exp(depth):
    p, leaf = depth_scene(depth)
    return oracle.voxel(p, leaf)


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
def test_skew(ctx, G):
    m = check(ctx, skew_split(G), 0.05, exp=_skew_exp())
    if G >= 4:
        assert (m.send.sum(0) == 0).any() and (m.send.sum(1) == 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
def test_exact_cut(ctx, G):
    """Cuts that the >= of the cut rule places (G = 2, 4, 8, 16): the device's cuts and send matrix are compared with the model's."""
    check(ctx, blocks(exact_cut_cloud(), G), 0.05, exp=_exact_exp())


@pytest.mark.gpu
@pytest.mark.parametrize("depth", DEPTHS)
@pytest.mark.parametrize("G", GS)
def test_octree_depths(ctx, G, depth):
    p, leaf = depth_scene(depth)
    check(ctx, blocks(p, G), leaf, exp=_depth_exp(depth))


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
def test_depth_22_is_rejected(ctx, G):
    p = boundary_cloud(50, 2100.0, seed=22)
    hs = [ctx.cloud_upload(q) for q in blocks(p, G)]
    expect_error(ctx, UNSUPPORTED, lambda: ctx.debug_voxel_distributed(hs, 0.001), launches=sum(len(q) > 0 for q in blocks(p, G)))
    for h in hs:
        ctx.cloud_free(h)


@pytest.mark.gpu
def test_shortcut_in_every_owner_range(ctx):
    """Two owner ranges of > 100k points each with strictly increasing codes under the global box: both take vox_single_kernel."""
    p = shortcut_cloud()
    locals_ = blocks(p, 2)
    hs = [ctx.cloud_upload(q) for q in locals_]
    before = ctx.voxel_shortcuts()
    got = run_handles(ctx, hs, 0.2)
    assert ctx.voxel_shortcuts() - before == 2
    for h in hs:
        ctx.cloud_free(h)
    check(ctx, locals_, 0.2, got=got)


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
def test_empty_ranks(ctx, G):
    p = cross_rank_cloud()[:5000]
    empty = p[:0]
    hs = [ctx.cloud_upload(empty) for _ in range(G)]
    out, cuts, send = run_handles(ctx, hs, 0.05)
    assert len(out) == 0 and not cuts.any() and not send.any()
    for h in hs:
        ctx.cloud_free(h)
    exp = oracle.voxel(p, 0.05)
    for where in (0, G - 1):
        locals_ = [p if r == where else empty for r in range(G)]
        m = check(ctx, locals_, 0.05, exp=exp)
        assert m.send.sum(1)[where] == len(p)


# ---------------------------------------------------------------------------------------------------------------- GPU: rejections
@pytest.mark.gpu
def test_rank_count_and_leaf_are_checked(ctx):
    hs = [ctx.cloud_upload(q) for q in blocks(cross_rank_cloud()[:1700], 17)]
    expect_error(ctx, UNSUPPORTED, lambda: ctx.debug_voxel_distributed(hs, 0.05), launches=0)
    for leaf in (0.0, -0.05, float("nan")):
        expect_error(ctx, INVALID, lambda: ctx.debug_voxel_distributed(hs[:4], leaf), launches=0)
    for h in hs:
        ctx.cloud_free(h)


def _nan_at(p, i):
    q = p.copy()
    q[i, 1] = np.nan
    return q


@pytest.mark.gpu
@pytest.mark.parametrize("G", GS)
def test_nan_on_one_rank_is_rejected_before_any_key(ctx, G):
    """One NaN on exactly one rank: every rank decides on the reduced non-finite flag, so the call fails after the extrema alone."""
    locals_ = blocks(cross_rank_cloud()[:8000], G)
    for r in range(G):
        bad = [_nan_at(q, len(q) // 2) if s == r else q for s, q in enumerate(locals_)]
        hs = [ctx.cloud_upload(q) for q in bad]
        e = expect_error(ctx, UNSUPPORTED, lambda: ctx.debug_voxel_distributed(hs, 0.05), launches=G)
        assert "non-finite" in str(e), r
        for h in hs:
            ctx.cloud_free(h)


def nonfinite_clouds():
    p = cross_rank_cloud()[:6000].copy()
    pinf, ninf = p.copy(), p.copy()
    pinf[4321, 0] = np.inf
    ninf[17, 2] = -np.inf
    allnan = p.copy()
    allnan[:, :3] = np.nan
    return [("+inf", pinf), ("-inf", ninf), ("all-NaN", allnan)]


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 3, 8])
def test_nonfinite_matches_the_serial_error(ctx, G):
    import lt_mapper_b200 as ltr
    for name, p in nonfinite_clouds():
        h = ctx.cloud_upload(p)
        with pytest.raises(ltr.LtrError) as serial_err:
            ctx.voxel_centroid(h, 0.05)
        ctx.cloud_free(h)
        hs = [ctx.cloud_upload(q) for q in blocks(p, G)]
        expect_error(ctx, serial_err.value.code, lambda: ctx.debug_voxel_distributed(hs, 0.05), launches=G)
        for h in hs:
            ctx.cloud_free(h)


def upper_face_cloud():
    """Finite points, one of them on the upper x face of the box: 4096 m from the minimum at leaf 1, where the f32 pad of the maximum
    rounds away, so its key is 2^12 = 2^depth and it falls outside the octree (ltr_voxel_centroid and the oracle reject the cloud)."""
    p = clustered(3000, 1.0, 100.0, seed=71, origin=10.0)
    p[5, 0], p[2000, 0] = 0.0, 4096.0
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 2, 5, 16])
def test_point_outside_the_box_is_rejected_on_every_rank(ctx, G):
    """Only the rank holding the point sees it outside; the outside count travels with the histogram sum, so every rank rejects, and
    its out-of-range code is not binned."""
    import lt_mapper_b200 as ltr
    p = upper_face_cloud()
    h = ctx.cloud_upload(p)
    with pytest.raises(ltr.LtrError) as serial_err:
        ctx.voxel_centroid(h, 1.0)
    ctx.cloud_free(h)
    hs = [ctx.cloud_upload(q) for q in blocks(p, G)]
    e = expect_error(ctx, serial_err.value.code, lambda: ctx.debug_voxel_distributed(hs, 1.0))
    assert "outside the octree" in str(e)
    for h in hs:
        ctx.cloud_free(h)


# ---------------------------------------------------------------------------------------------------------------- GPU: NCCL, world 1
@pytest.fixture(scope="module")
def comm(ctx):
    import torch  # noqa: F401 -- loads the libnccl.so.2 that nccl_comm.cu dlopens
    from lt_mapper_b200 import binding
    L = binding.lib()
    v = ctypes.c_int32()
    if L.ltr_nccl_version(ctypes.byref(v)) != 0:
        pytest.skip("libnccl.so.2 cannot be loaded")
    uid = (ctypes.c_uint8 * 128)()
    assert L.ltr_nccl_unique_id(uid) == 0
    c = ctypes.c_int32()
    ctx._ck(L.ltr_nccl_init(ctx._h, uid, 0, 1, ctypes.byref(c)))
    yield c.value
    ctx._ck(L.ltr_nccl_destroy(ctx._h, c.value))


def merged(ctx, comm, h, leaf):
    from lt_mapper_b200 import binding
    o = ctypes.c_int32()
    ctx._ck(binding.lib().ltr_nccl_voxel_centroid_merged(ctx._h, comm, h, leaf, ctypes.byref(o)))
    got = ctx.cloud_download(o.value).copy()
    ctx.cloud_free(o.value)
    return got


@pytest.mark.gpu
def test_nccl_world1_equals_the_serial_voxeliser(ctx, comm):
    scenes = [(cross_rank_cloud(), 0.05), (skew_cloud(), 0.05), (exact_cut_cloud(), 0.05), (shortcut_cloud(), 0.2)]
    scenes += [depth_scene(d) for d in DEPTHS]
    for p, leaf in scenes:
        h = ctx.cloud_upload(p)
        assert np.array_equal(bits(merged(ctx, comm, h, leaf)), bits(serial(ctx, p, leaf))), (len(p), leaf)
        ctx.cloud_free(h)
    p = cross_rank_cloud()
    h = ctx.cloud_upload(p)
    v = ctx.cloud_slice(h, 1234, 30_000)                                # a strided view at a non-zero offset
    assert np.array_equal(bits(merged(ctx, comm, v, 0.05)), bits(oracle.voxel(p[1234:30_000], 0.05)))
    ctx.cloud_free(v)
    e = ctx.cloud_upload(p[:0])
    assert len(merged(ctx, comm, e, 0.05)) == 0
    for x in (e, h):
        ctx.cloud_free(x)


@pytest.mark.gpu
def test_nccl_world1_rejects_nonfinite(ctx, comm):
    """All-NaN, +inf and -inf clouds fail with ltr_voxel_centroid's code after the extrema alone, and return their scratch."""
    for name, p in nonfinite_clouds():
        h = ctx.cloud_upload(p)
        e = expect_error(ctx, UNSUPPORTED, lambda: merged(ctx, comm, h, 0.05), launches=1)
        assert "non-finite" in str(e), name
        ctx.cloud_free(h)
    h = ctx.cloud_upload(upper_face_cloud())
    expect_error(ctx, UNSUPPORTED, lambda: merged(ctx, comm, h, 1.0))
    ctx.cloud_free(h)


# ---------------------------------------------------------------------------------------------------------------- CPU self-checks
def test_selfcheck_pipeline_blocks_leave_ranks_empty(small_pair):
    K = small_pair[0].K
    assert K == 6
    assert sum(K * (r + 1) // 8 == K * r // 8 for r in range(8)) == 2


def test_selfcheck_cross_rank_voxels():
    """Most voxels have points on two or more source ranks for every G >= 2."""
    p = cross_rank_cloud()
    for G in GS[1:]:
        code = morton(p, define_box(p, 0.05))
        rank = np.repeat(np.arange(G), [len(q) for q in blocks(p, G)])
        pairs = np.unique(np.stack([code, rank.astype(np.uint64)], 1), axis=0)
        _, per_voxel = np.unique(pairs[:, 0], return_counts=True)
        assert (per_voxel >= 2).mean() > 0.6, G
        assert np.median(np.unique(code, return_counts=True)[1]) >= 2


def test_selfcheck_skew():
    """One prefix bin holds >= 60 % of the points, several cuts land on it, and from G = 4 on some ranks receive nothing and one rank
    sends nothing."""
    for G in GS:
        m = dist_model(skew_split(G), 0.05)
        assert m.hg.max() >= 0.6 * m.hg.sum() and m.shift > 0
        if G >= 4:
            assert len(np.unique(m.cuts)) < len(m.cuts), G
            assert (m.send.sum(0) == 0).any() and (m.send.sum(1) == 0).any(), G
            assert (m.send.sum(0) > 0).sum() >= 2, G


def test_selfcheck_exact_cut():
    """For G = 2, 4, 8 and 16 some cut falls where cum * G == total * (j + 1) holds exactly, followed by empty bins: a strict comparison
    would move that cut and change the send matrix."""
    for G in GS:
        locals_ = blocks(exact_cut_cloud(), G)
        m, ms = dist_model(locals_, 0.05), dist_model(locals_, 0.05, strict=True)
        cum = np.cumsum(m.hg)
        total = int(cum[-1])
        exact = [j for j in range(G - 1) if (cum * G == total * (j + 1)).any()]
        if G in (2, 4, 8, 16):
            assert exact and not np.array_equal(m.cuts, ms.cuts) and not np.array_equal(m.send, ms.send), G
        else:
            assert not exact, G


def test_selfcheck_octree_depths():
    for depth in DEPTHS:
        p, leaf = depth_scene(depth)
        m = dist_model([p], leaf)
        assert m.depth == depth, (depth, m.depth)
        assert m.nbins == 1 << min(12, 3 * depth) and m.shift == max(0, 3 * depth - 12)
    assert dist_model([depth_scene(1)[0]], 1.0).nbins == 8
    p = pair_cloud()
    for G in GS:
        m = dist_model(blocks(p, G), PAIR_LEAF)
        assert min(key_bits(17, len(o)) for o in owner_ranges(blocks(p, G), m)) > 64, G   # every owner range takes the pair sort
    assert define_box(boundary_cloud(50, 2100.0, seed=22), 0.001)[2] == 22


def test_selfcheck_shortcut_ranges():
    p = shortcut_cloud()
    locals_ = blocks(p, 2)
    m = dist_model(locals_, 0.2)
    for o in owner_ranges(locals_, m):
        code = morton(o, m.box)
        assert len(o) >= SHORTCUT_MIN and (code[1:] > code[:-1]).all() and key_bits(m.depth, len(o)) <= 64


def test_selfcheck_upper_face_point_is_outside():
    p = upper_face_cloud()
    lo, res, depth = define_box(p, 1.0)
    assert depth == 12 and lo[0] == 0.0 and (float(p[:, 0].max()) - lo[0]) / res == 1 << depth
    assert ((p[:, 0].astype(np.float64) - lo[0]) / res >= 1 << depth).sum() == 1
    with pytest.raises(ValueError):
        oracle.voxel(p, 1.0)


def test_selfcheck_model_counts_every_point():
    for G in GS:
        locals_ = blocks(cross_rank_cloud(), G)
        m = dist_model(locals_, 0.05)
        assert m.send.sum(1).tolist() == [len(q) for q in locals_]
        assert (np.diff(m.cuts.astype(np.int64)) >= 0).all() and len(m.cuts) == G - 1
        sizes = m.send.sum(0)
        assert sizes.max() - sizes.min() <= max(m.hg.max(), 1), G          # ranges of nearly equal population
