"""Voxeliser (util.cu: Morton keys, the stable radix sort with and without a separate index, per-voxel f32 sums, the one-point-per-voxel
shortcut) and the stable partition, at the shapes the pipeline never reaches, bit for bit against oracle.voxel / numpy.

The inputs are built so that the f32 sums depend on the order of summation: voxels of 2 to 50 points in shuffled insertion order,
intensities of about 1e4 and 1e-3 mixed inside a voxel and coordinates about 1e3 m from the origin.  A sort that loses stability
changes bits.  The tests without the gpu mark check on the CPU that each input takes the path its GPU test claims.
"""
import math

import numpy as np
import pytest

import oracle

F32 = np.float32
FLT_EPS = float(np.finfo(F32).eps)
RS_TILE = 4096                   # kRsTile: keys per radix-sort tile
KEY_STRIDE = 255                 # kVoxKeyStride: points per key block (blocks of 256 threads overlap by one point)
SHORTCUT_MIN = 100000            # kVoxShortcutMin
PAIR_LEAF = 0.01


# ---------------------------------------------------------------------------------------------------------------- references
def define_box(p, leaf):
    """Python copy of define_box (util.cu): (box minimum per axis, resolution, octree depth)."""
    mn, mx = p[:, :3].min(0), p[:, :3].max(0)
    res = float(F32(leaf))
    lo = mn.astype(np.float64)
    hi = (mx + F32(FLT_EPS * 512)).astype(F32).astype(np.float64)
    lo, hi = np.minimum(lo, hi), np.maximum(np.minimum(lo, hi), hi)
    mk = np.ceil((hi - lo - FLT_EPS) / res)
    lg = math.log(max(int(mk.max()), 2)) / math.log(2.0)
    depth = max(min(32, math.ceil(lg - FLT_EPS)), 0)
    over = ((1 << depth) * res - (hi - lo)) / 2.0
    return np.where(over > FLT_EPS, lo - over, lo), res, depth


def key_bits(depth, n):
    """Bits of Morton code + point index; voxel_view packs both into one 64-bit key iff this is <= 64."""
    idx_bits = 1
    while idx_bits < 32 and (1 << idx_bits) < n:
        idx_bits += 1
    return 3 * depth + idx_bits


def morton(p, box):
    lo, res, depth = box
    kk = ((p[:, :3].astype(np.float64) - lo) / res).astype(np.uint64)
    code = np.zeros(len(p), np.uint64)
    for b in range(depth):
        for a in range(3):
            code |= ((kk[:, a] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + 2 - a)
    return code


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------- inputs
def clustered(n, leaf, extent, seed, origin=1000.0):
    """n points in clusters of 2..50 points, each far smaller than a voxel, in shuffled order; intensities ~1e4 and ~1e-3 mixed."""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(2, 51, n // 2 + 1)
    sizes = sizes[: np.searchsorted(np.cumsum(sizes), n) + 1]
    sizes[-1] -= sizes.sum() - n
    centres = origin + rng.uniform(0, 1, (len(sizes), 3)) * extent
    xyz = np.repeat(centres, sizes, 0) + rng.uniform(-0.25, 0.25, (n, 3)) * leaf
    inten = np.where(rng.random(n) < 0.5, rng.uniform(1e4, 2e4, n), rng.uniform(1e-3, 2e-3, n))
    out = np.concatenate([xyz, inten[:, None]], 1).astype(F32)
    return out[rng.permutation(n)]


def pair_cloud():
    """About 300k points over 1.3 km at leaf 0.01: depth 17, 51 code bits + 19 index bits > 64 -> (key, index) pair sort."""
    return clustered(300_000, PAIR_LEAF, 1300.0, seed=1)


def boundary_cloud(n, extent, seed):
    """n points at leaf 0.001 over `extent` metres of x (the long axis, so both x halves of the box are used), a few sharing a voxel."""
    rng = np.random.default_rng(seed)
    xyz = 1000.0 + rng.uniform(0, 1, (n, 3)) * [extent, 3.0, 3.0]
    xyz[0, 0], xyz[1, 0] = 1000.0, 1000.0 + extent
    if n > 8:
        xyz[3:7] = xyz[2] + rng.uniform(0, 2e-4, (4, 3))
    inten = np.where(rng.random(n) < 0.5, 1.5e4, 1.7e-3) * rng.uniform(1, 2, n)
    return np.concatenate([xyz, inten[:, None]], 1).astype(F32)[rng.permutation(n)]


def one_voxel_cloud():
    """1M points inside one voxel plus two outliers that set the box: one thread sums a run of 1M points."""
    rng = np.random.default_rng(3)
    xyz = rng.uniform(50.2, 50.8, (1_000_000, 3))
    inten = np.where(rng.random(1_000_000) < 0.5, rng.uniform(1e4, 2e4, 1_000_000), rng.uniform(1e-3, 2e-3, 1_000_000))
    pts = np.concatenate([xyz, inten[:, None]], 1)
    return np.concatenate([[[0, 0, 0, 1]], pts[:600_000], [[100, 100, 100, 2]], pts[600_000:]]).astype(F32)


def one_per_voxel(n, extent, leaf, seed):
    """A voxelised cloud: (about) one point per voxel, in octree order."""
    rng = np.random.default_rng(seed)
    pts = np.concatenate([rng.uniform(0, extent, (n, 3)) + 500.0, rng.uniform(0, 1, (n, 1))], 1).astype(F32)
    return oracle.voxel(pts, leaf)


SEAMS = [(31, 32), (254, 255), (255, 256), (286, 287), (509, 510)]     # warp and block seams of the 255-point key blocks
SHORTCUT_LEAF = 0.2


def shortcut_variants():
    """The untouched voxelised cloud and, one at a time, an adjacent pair swapped at a seam (or at the end), or a point moved into
    its predecessor's voxel (equal codes: not strictly increasing)."""
    v = one_per_voxel(300_000, 200.0, SHORTCUT_LEAF, seed=9)
    out = [("untouched", v, None)]
    for i, j in SEAMS + [(len(v) - 2, len(v) - 1)]:
        s = v.copy()
        s[[i, j]] = s[[j, i]]
        out.append((f"swap {i},{j}", s, j))            # the first code that is not above its predecessor
    for i in (32, 256):
        s = v.copy()
        s[i, :3] = s[i - 1, :3]
        out.append((f"equal code at {i}", s, i))
    return out


SIZES = [1, 2, 3, 255, 256, 4095, 4096, 4097, 99_999, 100_000, 1 << 20, (1 << 20) + 1, 3 * (1 << 20) + 5]


def sized_cloud(n):
    return clustered(n, 0.05, 100.0, seed=n)


KF_LEAF = PAIR_LEAF


def keyframes():
    """Ragged keyframes for ltr_voxel_centroid_per_keyframe, all at leaf 0.01: the 150k one-per-voxel keyframe takes the shortcut at
    a non-zero offset, the 300k one the pair sort."""
    parts = [np.zeros((0, 4), F32), clustered(1, KF_LEAF, 1.0, 21), clustered(3, KF_LEAF, 1.0, 22), clustered(5000, KF_LEAF, 10.0, 23),
             np.zeros((0, 4), F32), one_per_voxel(150_000, 40.0, KF_LEAF, seed=24), pair_cloud(), clustered(7, KF_LEAF, 1.0, 25)]
    return parts


# ---------------------------------------------------------------------------------------------------------------- GPU tests
@pytest.fixture(scope="module")
def ctx():
    import lt_mapper_b200 as ltr
    c = ltr.Context()
    yield c
    c.close()


def voxelise(ctx, p, leaf):
    h = ctx.cloud_upload(p)
    before = ctx.voxel_shortcuts()
    o = ctx.voxel_centroid(h, leaf)
    got = ctx.cloud_download(o).copy()
    shortcuts = ctx.voxel_shortcuts() - before
    ctx.cloud_free(h)
    ctx.cloud_free(o)
    return got, shortcuts


def check_voxel(ctx, p, leaf):
    got, shortcuts = voxelise(ctx, p, leaf)
    exp = oracle.voxel(p, leaf)
    assert got.shape == exp.shape and np.array_equal(bits(got), bits(exp))
    return shortcuts


@pytest.mark.gpu
def test_pair_sort_path(ctx):
    p = pair_cloud()
    assert check_voxel(ctx, p, PAIR_LEAF) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("n,extent", [(2, 1500.0), (16, 600.0), (17, 600.0)])
def test_packing_boundary(ctx, n, extent):
    """Depth 21 with 2 points packs into exactly 64 bits; depth 20 with 16 points packs (64 bits), with 17 it takes the pair sort."""
    check_voxel(ctx, boundary_cloud(n, extent, seed=n), 0.001)


@pytest.mark.gpu
def test_depth_22_is_rejected(ctx):
    import lt_mapper_b200 as ltr
    p = boundary_cloud(50, 2100.0, seed=22)
    with pytest.raises(ValueError):
        oracle.voxel(p, 0.001)
    h = ctx.cloud_upload(p)
    base = ctx.memory_stats()[0]
    with pytest.raises(ltr.LtrError) as e:
        ctx.voxel_centroid(h, 0.001)
    assert e.value.code == -3 and ctx.memory_stats()[0] == base
    ctx.cloud_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_sizes(ctx, n):
    check_voxel(ctx, sized_cloud(n), 0.05)


@pytest.mark.gpu
def test_one_voxel_of_a_million_points(ctx):
    got, _ = voxelise(ctx, one_voxel_cloud(), 1.0)
    exp = oracle.voxel(one_voxel_cloud(), 1.0)
    assert len(exp) == 3 and np.array_equal(bits(got), bits(exp))


@pytest.mark.gpu
def test_shortcut_detector_at_block_and_warp_seams(ctx):
    for name, p, first_bad in shortcut_variants():
        assert check_voxel(ctx, p, SHORTCUT_LEAF) == (1 if first_bad is None else 0), name


@pytest.mark.gpu
def test_voxel_centroid_per_keyframe(ctx):
    import lt_mapper_b200 as ltr
    parts = keyframes()
    off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    ss = ctx.scanset_upload(np.concatenate(parts), off)
    before = ctx.voxel_shortcuts()
    out = ctx.voxel_centroid_per_keyframe(ss, KF_LEAF)
    assert ctx.voxel_shortcuts() - before == 1
    pts, noff = ctx.scanset_download(out)
    exp = [oracle.voxel(p, KF_LEAF) if len(p) else np.zeros((0, 4), F32) for p in parts]
    assert np.array_equal(noff, np.concatenate([[0], np.cumsum([len(e) for e in exp])]))
    for k, e in enumerate(exp):
        assert np.array_equal(bits(pts[noff[k]:noff[k + 1]]), bits(e)), k
    ctx.scanset_free(out)
    ctx.scanset_free(ss)
    bad = [p.copy() for p in parts]
    bad[3][1234, 2] = np.nan
    ss = ctx.scanset_upload(np.concatenate(bad), off)
    base = ctx.memory_stats()[0]
    with pytest.raises(ltr.LtrError) as e:
        ctx.voxel_centroid_per_keyframe(ss, KF_LEAF)
    assert e.value.code == -3 and ctx.memory_stats()[0] == base
    ctx.scanset_free(ss)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 255, 257, 2047, 2049, (1 << 20) + 3, (1 << 25) + 7])
def test_stable_partition(ctx, n):
    """ltr_apply_partition (stable_partition_by_flag) around the 256-thread block and the 2048-point tile, and at 2^25 + 7 points."""
    rng = np.random.default_rng(n)
    p = rng.standard_normal((n, 4), F32)
    h = ctx.cloud_upload(p)
    for name, f in (("zeros", np.zeros(n, np.uint8)), ("ones", np.ones(n, np.uint8)), ("alternating", (np.arange(n) & 1).astype(np.uint8)),
                    ("random", (rng.random(n) < 0.3).astype(np.uint8))):
        ctx.flags_upload(h, f)
        s, d = ctx.apply_partition(h)
        assert np.array_equal(bits(ctx.cloud_download(s)), bits(p[f == 0])), name
        assert np.array_equal(bits(ctx.cloud_download(d)), bits(p[f == 1])), name
        ctx.cloud_free(s)
        ctx.cloud_free(d)
    ctx.cloud_free(h)


# ---------------------------------------------------------------------------------------------------------------- CPU self-checks
def test_selfcheck_pair_cloud_takes_the_pair_sort():
    p = pair_cloud()
    _, _, depth = define_box(p, PAIR_LEAF)
    assert depth == 17 and key_bits(depth, len(p)) == 70
    assert np.median(np.unique(morton(p, define_box(p, PAIR_LEAF)), return_counts=True)[1]) >= 2   # mostly multi-point voxels


def test_selfcheck_packing_boundary():
    for n, extent, depth, nbits in ((2, 1500.0, 21, 64), (16, 600.0, 20, 64), (17, 600.0, 20, 65)):
        p = boundary_cloud(n, extent, seed=n)
        box = define_box(p, 0.001)
        assert box[2] == depth and key_bits(depth, n) == nbits, n
        code = morton(p, box)
        top = np.uint64(1) << np.uint64(3 * depth - 1)
        assert (code & top).any() and not (code & top).all(), n          # both x halves: a key that drops the top bit reorders
        if nbits == 65:
            assert not np.array_equal(np.argsort(code, kind="stable"), np.argsort(code & (top - np.uint64(1)), kind="stable"))
    assert define_box(boundary_cloud(50, 2100.0, seed=22), 0.001)[2] == 22


def test_selfcheck_sizes():
    for n in SIZES:
        p = sized_cloud(n)
        assert len(p) == n and key_bits(define_box(p, 0.05)[2], n) <= 64
    tiles = [(n + RS_TILE - 1) // RS_TILE for n in ((1 << 20), (1 << 20) + 1)]
    assert 256 * tiles[0] <= 65536 < 256 * tiles[1]         # single-block scan of the digit matrix vs exclusive_scan_u32


def test_selfcheck_one_voxel_cloud():
    p = one_voxel_cloud()
    code = morton(p, define_box(p, 1.0))
    assert len(np.unique(code)) == 3 and np.unique(code, return_counts=True)[1].max() == 1_000_000


def test_selfcheck_shortcut_variants():
    """The untouched cloud has strictly increasing codes; every variant breaks that at exactly the point it meant to."""
    for name, p, first_bad in shortcut_variants():
        box = define_box(p, SHORTCUT_LEAF)
        code = morton(p, box)
        assert len(p) >= SHORTCUT_MIN and key_bits(box[2], len(p)) <= 64
        bad = np.flatnonzero(~(code[1:] > code[:-1])) + 1
        assert bad.tolist() == ([] if first_bad is None else [first_bad]), name


def test_selfcheck_keyframes():
    parts = keyframes()
    assert [len(p) for i, p in enumerate(parts) if i != 5] == [0, 1, 3, 5000, 0, 300_000, 7] and 149_900 < len(parts[5]) <= 150_000
    v = parts[5]
    box = define_box(v, KF_LEAF)
    code = morton(v, box)
    assert (code[1:] > code[:-1]).all()
    assert key_bits(define_box(parts[6], KF_LEAF)[2], len(parts[6])) > 64
