"""kNN labelling (knn.cu) on its dense-grid path at the shapes and edges the pipeline never reaches.

Covered: every k of the 16-slot top list, averages exactly on the threshold, neighbours at the reach across one and two cell faces,
the x1.25 cell growth, degenerate targets, queries outside the grid (up to infinite distances), awkward ltr_knn_diff set-ups, the
benchmark's shape and non-finite targets.  References: oracle.knn_partition, bit for bit, for ltr_knn_diff, and for
ltr_knn_split_cloud labels built from oracle.knn_dists the way the reference builds them (Session.cpp:592-596).  The tests without
the gpu mark check on the CPU that each input really takes the path its GPU test claims.
"""
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import oracle

F32 = np.float32
I4 = np.eye(4)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_CELLS = 536870912.0          # build_grid's bound on the dense grid (2^29 cells)
THRS = (1e-4, 0.01, 0.04, 1.0, 25.0)


# ---------------------------------------------------------------------------------------------------------------- references
def grid_geometry(t, k, thr):
    """Python copy of build_grid (knn.cu): (cell side, grid origin per axis, number of x1.25 growth steps)."""
    mn, mx = t[:, :3].min(0), t[:, :3].max(0)
    cell = math.sqrt(k * float(F32(thr))) * 1.001 + 1e-6
    steps = 0
    while True:
        cells = 1.0
        for d in range(3):
            cells *= math.floor((float(mx[d]) - float(mn[d])) / cell) + 3.0
        if cells <= MAX_CELLS:
            break
        cell *= 1.25
        steps += 1
    return cell, mn.astype(np.float64) - cell, steps


def ref_labels(q, t, k, thr):
    """1 = far: |(float)(sum_double of the k smallest squared distances) / float(k)| >= thr.  The double sum runs one column at a
    time, in order, as std::accumulate does (np.sum over the axis is pairwise for k >= 8)."""
    d = oracle.knn_dists(q, t, k)
    s = np.zeros(len(q))
    for j in range(min(k, len(t))):
        s = s + d[:, j].astype(np.float64)
    with np.errstate(over="ignore"):                   # sums beyond FLT_MAX become inf, as (float)sum does
        avg = s.astype(F32) / F32(k)
    return (~(np.abs(avg) < F32(thr))).astype(np.uint8)


def check_kdtree(q, t, k, budget=20_000_000):
    """oracle.knn_dists (k-d tree) == brute force on as many queries as the budget of distance evaluations allows."""
    m = max(1, min(len(q), budget // max(len(t), 1)))
    sub = q[np.linspace(0, len(q) - 1, m).astype(np.int64)]
    assert np.array_equal(oracle.knn_dists(sub, t, k).view(np.uint32), oracle.knn_dists(sub, t, k, brute=True).view(np.uint32))


def xyzi(p, first_id=0):
    """(n, 3) -> (n, 4) float32 with the point's number as intensity."""
    p = np.asarray(p, np.float64).reshape(-1, 3)
    return np.concatenate([p, np.arange(first_id, first_id + len(p))[:, None]], 1).astype(F32)


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------- inputs
def density_scene(thr, seed=0, nq=20000):
    """Four slabs of target density 100, 10, 1 and 0.1 points per unit^3 side by side, queries uniform over all of them plus a
    quarter jittered copies of targets; lengths scaled by sqrt(thr), so that every k from 1 to 16 finds near and far points."""
    rng = np.random.default_rng(seed)
    parts, x0 = [], 0.0
    for rho, length in ((100, 2.0), (10, 5.0), (1, 10.0), (0.1, 30.0)):
        n = int(rho * 100 * length)
        parts.append(rng.uniform(0, 1, (n, 3)) * [length, 10, 10] + [x0, 0, 0])
        x0 += length
    t = np.concatenate(parts)
    q = rng.uniform(0, 1, (nq, 3)) * [x0, 10, 10]
    q[: nq // 4] = t[rng.integers(0, len(t), nq // 4)] + rng.normal(0, 0.1, (nq // 4, 3))
    s = math.sqrt(thr)
    return xyzi(q * s), xyzi(t * s, 1000000)


def threshold_sets(k, seed):
    """Hand-built distance sets: (squared distances, thr, expected label, what) with every squared distance exact in f32.
    Distances are multiples of 2^-5 below 128, so that they stay exact 3e5 m from the origin and their squares are exact."""
    rng = np.random.default_rng(seed)
    out = []

    def correct(d):
        return F32(F32(math.fsum(d)) / F32(k))          # exact double sum (multiples of 2^-10) -> f32 -> / k in f32

    m = rng.integers(1, 4096, k)
    d = (m.astype(np.float64) / 32) ** 2
    c = correct(d)
    out.append((m, c, 1, "avg == thr is far (strict <)"))
    out.append((m, np.nextafter(c, F32(np.inf)), 0, "thr one ulp above avg is near"))
    # both polarities where they occur (one of them may be rare or impossible for a given k)
    need = {(what, above) for what in (["f32 running sum"] if k >= 3 else []) + (["f64 divide"] if k & (k - 1) else [])
            for above in (False, True)}                # dividing by a power of two is exact either way
    found = {}
    for _ in range(20000):
        if need <= set(found):
            break
        m = rng.integers(1, 4096, k)
        d = (m.astype(np.float64) / 32) ** 2
        c = correct(d)
        run = F32(0)
        for v in d:
            run = F32(run + F32(v))
        for what, w in (("f64 divide", F32(math.fsum(d) / k)), ("f32 running sum", F32(run / F32(k)))):
            key = (what, bool(c > w))
            if w == c or key in found:
                continue
            # thr between the two candidates: the correct mean decides, the wrong one would decide the other way
            found[key] = (m, c, 1, f"{what}: {w} < avg") if c > w else (m, np.nextafter(c, F32(np.inf)), 0, f"{what}: {w} > avg")
    assert {w for w, _ in need} <= {w for w, _ in found}, (k, need - set(found))
    return out + list(found.values())


AXES = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64)


def axis_targets(centre, m):
    """Point j at distance m[j] / 32 from centre along axis direction j % 6."""
    return centre + AXES[np.arange(len(m)) % 6] * (np.asarray(m, np.float64)[:, None] / 32)


def reach_scene(k, thr, seed, n=60000):
    """Queries with k - 1 targets on top of them and one more at a squared distance straddling k*thr (by the f32 spacing of the
    coordinates, a few parts in 1e5), along an axis (across one cell face) or diagonally in x and y (across two).  Half of the
    queries sit on cell faces of build_grid's grid (to within 0..2 ulps), half anywhere; queries are 6 cells apart so that each
    sees only its own targets."""
    rng = np.random.default_rng(seed)
    R = math.sqrt(k * float(F32(thr)))
    cell = R * 1.001 + 1e-6                           # no growth at these extents (checked on the CPU below)
    lo = np.full(3, 1.0)                              # two anchor targets fix the box: mn = lo, hence origin = lo - cell
    origin = lo - cell
    side = int(round(n ** (1 / 3))) + 1
    lattice = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n]
    faces = origin + (6 * lattice + 3) * cell                      # face 6j + 3 of every axis
    on_face = rng.random(n) < 0.5
    q = np.where(on_face[:, None], faces, faces + rng.uniform(0.05, 0.95, (n, 3)) * cell).astype(F32)
    nudge = rng.integers(-2, 3, (n, 3))                            # 0..2 ulps off the face
    towards = np.where(nudge > 0, F32(np.inf), F32(-np.inf))
    for step in (1, 2):
        q = np.where(on_face[:, None] & (np.abs(nudge) >= step), np.nextafter(q, towards), q)
    diag = rng.random(n) < 0.3
    axis = rng.integers(0, 6, n)
    dirn = np.where(diag[:, None], np.array([-1.0, -1.0, 0.0]) / math.sqrt(2), AXES[axis])
    r = R * (1 + rng.uniform(-2e-5, 2e-5, n))
    far_pt = (q.astype(np.float64) + dirn * r[:, None]).astype(F32)
    tgt = [np.repeat(q, k - 1, 0), far_pt, np.array([lo, lo + (6 * side + 2) * cell], F32)]
    return xyzi(q), xyzi(np.concatenate(tgt), 10_000_000), cell


def growth_scene(seed=11, nt=1_000_000, nq=200_000):
    """About 1M targets over 20 km x 20 km x 40 m: k = 1, thr = 1e-4 would need ~10^16 cells of side 1 cm."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(0, 1, (nt, 3)) * [20000, 20000, 40] - [10000, 10000, 20]
    q = rng.uniform(0, 1, (nq, 3)) * [20000, 20000, 40] - [10000, 10000, 20]
    q[: nq // 2] = t[rng.integers(0, nt, nq // 2)] + rng.normal(0, 0.006, (nq // 2, 3))
    return xyzi(q), xyzi(t, 10_000_000)


def outside_scene(seed=4):
    rng = np.random.default_rng(seed)
    t = xyzi(rng.uniform(0, 1, (4000, 3)), 100000)
    k, thr = 2, 0.005
    cell, origin, _ = grid_geometry(t, k, thr)
    lo, hi = t[:, :3].min(0).astype(np.float64), t[:, :3].max(0).astype(np.float64)
    q = []
    for d in range(3):
        for s in (-1, 1):
            for f in np.arange(0.5, 3.01, 0.25):
                p = rng.uniform(lo, hi, (40, 3))
                p[:, d] = (hi[d] + f * cell) if s > 0 else (lo[d] - f * cell)
                q.append(p)
    q = np.concatenate(q)
    special = [[1e19, 0.5, 0.5], [-1e19, 0.5, 0.5], [0.5, 1e19, 0.5], [0.5, 0.5, -1e19], [1e19, 1e19, 1e19], [-1e19, 1e19, -1e19],
               [1e30, 0.5, 0.5], [-1e30, 0.5, 0.5], [0.5, -1e30, 0.5], [0.5, 0.5, 1e30], [1e30, -1e30, 1e30],
               [-0.0, -0.0, -0.0], [-0.0, 0.5, 0.5], [0.5, -0.0, 0.0]]
    return xyzi(np.concatenate([q, special])), t, k, thr


# ---------------------------------------------------------------------------------------------------------------- GPU tests
@pytest.fixture(scope="module")
def ctx():
    import lt_mapper_b200 as ltr
    c = ltr.Context()
    yield c
    c.close()


def run_split(ctx, q, t, k, thr):
    qh, th = ctx.cloud_upload(q), ctx.cloud_upload(t)
    nh, fh = ctx.knn_split_cloud(qh, th, k, thr)
    near, far = ctx.cloud_download(nh).copy(), ctx.cloud_download(fh).copy()
    for h in (qh, th, nh, fh):
        ctx.cloud_free(h)
    return near, far


def check_split(ctx, q, t, k, thr, lab):
    near, far = run_split(ctx, q, t, k, thr)
    assert np.array_equal(bits(near), bits(q[lab == 0])) and np.array_equal(bits(far), bits(q[lab == 1])), (k, thr)


def check_diff(ctx, q, t, k, thr, lab=None):
    """ltr_knn_diff, one keyframe with the identity pose, against oracle.knn_partition (and its labels against `lab`)."""
    ss = ctx.scanset_upload(q, [0, len(q)])
    ps = ctx.poses_upload(I4[None], I4[None])
    th = ctx.cloud_upload(t)
    co, di = ctx.knn_diff(ss, ps, th, k, thr)
    olab, eco, edi = oracle.knn_partition(q, I4, I4, t, k, thr)
    if lab is not None:
        assert np.array_equal(olab, lab), (k, thr)
    cp, _ = ctx.scanset_download(co)
    dp, _ = ctx.scanset_download(di)
    assert np.array_equal(bits(cp), bits(eco)) and np.array_equal(bits(dp), bits(edi)), (k, thr)
    for s in (ss, co, di):
        ctx.scanset_free(s)
    ctx.poses_free(ps)
    ctx.cloud_free(th)


def check_both(ctx, q, t, k, thr, brute=True):
    lab = ref_labels(q, t, k, thr)
    if brute:
        check_kdtree(q, t, k)
    check_split(ctx, q, t, k, thr, lab)
    check_diff(ctx, q, t, k, thr, lab)
    return lab


@pytest.mark.gpu
@pytest.mark.parametrize("thr", THRS)
@pytest.mark.parametrize("k", range(1, 17))
def test_every_k_on_the_grid_path(ctx, k, thr):
    q, t = density_scene(thr)
    lab = check_both(ctx, q, t, k, thr, brute=False)
    assert 0.1 < lab.mean() < 0.9


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0.0, 3e5])
@pytest.mark.parametrize("k", [1, 2, 3, 5, 7, 16])
def test_hand_built_thresholds(ctx, k, offset):
    """Query at (offset, offset, offset), exactly k targets on the axes.  avg == thr must be far, thr one ulp above near; where a
    double sum divided in f64, or a running f32 sum, gives a different mean, thr sits between the candidates."""
    centre = np.full(3, offset)
    for m, thr, expect, what in threshold_sets(k, seed=k):
        q, t = xyzi(centre), xyzi(axis_targets(centre, m), 10)
        assert np.array_equal(oracle.knn_dists(q, t, k)[0], np.sort(m / 32) ** 2)
        lab = check_both(ctx, q, t, k, float(thr))
        assert lab[0] == expect, (what, m, thr)


@pytest.mark.gpu
@pytest.mark.parametrize("k,thr", [(1, 0.01), (1, 1.0), (4, 0.04), (16, 0.01), (16, 1.0)])
def test_neighbours_at_the_reach_across_cell_faces(ctx, k, thr):
    q, t, _ = reach_scene(k, thr, seed=k)
    lab = check_both(ctx, q, t, k, thr)
    assert 0.2 < lab.mean() < 0.8


@pytest.mark.gpu
def test_grid_growth_on_a_20_km_map(ctx):
    q, t = growth_scene()
    lab = ref_labels(q, t, 1, 1e-4)
    check_split(ctx, q, t, 1, 1e-4, lab)
    assert 0.2 < lab.mean() < 0.8


DEGENERATE = ("flat", "collinear", "identical", "duplicated")


def degenerate_scene(kind, rng):
    if kind == "flat":
        t = np.concatenate([rng.uniform(-5, 5, (5000, 2)), np.full((5000, 1), 1.25)], 1)
    elif kind == "collinear":
        t = np.outer(rng.uniform(-20, 20, 5000), [0.6, 0.8, 0.0]) + [3, -2, 1]
    elif kind == "identical":
        t = np.tile([[1.5, -2.5, 0.75]], (100, 1))
    else:   # 64 copies of each of 1000 points: ties at the k-th distance
        t = np.repeat(rng.uniform(-5, 5, (1000, 3)), 64, 0)
    t = t.astype(F32).astype(np.float64)
    lo, hi = t.min(0) - 1, t.max(0) + 1
    q = rng.uniform(lo, hi, (3000, 3))
    q[:1000] = t[rng.integers(0, len(t), 1000)] + rng.normal(0, 0.15, (1000, 3))
    q[1000:1100] = t[rng.integers(0, len(t), 100)]                                  # exactly on a target
    return xyzi(q), xyzi(t, 100000)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", DEGENERATE)
@pytest.mark.parametrize("k,thr", [(2, 0.04), (16, 0.05), (16, 1.0)])
def test_degenerate_targets(ctx, kind, k, thr):
    q, t = degenerate_scene(kind, np.random.default_rng(DEGENERATE.index(kind)))
    lab = check_both(ctx, q, t, k, thr)
    assert 0 < lab.sum() < len(lab)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 5, 16])
def test_target_of_k_and_k_minus_one_points(ctx, k):
    """k points take the grid path, k - 1 the brute-force one; both must give the reference's labels."""
    rng = np.random.default_rng(k)
    pts = rng.uniform(-1, 1, (k, 3))
    q = rng.uniform(-2, 2, (5000, 3))
    q[:2000] = pts[rng.integers(0, k, 2000)] + rng.normal(0, 0.3, (2000, 3))
    for n in (k, k - 1):
        lab = check_both(ctx, xyzi(q), xyzi(pts[:n], 100), k, 1.5)
        assert 0 < lab.sum() < len(lab), n


@pytest.mark.gpu
def test_queries_outside_the_grid(ctx):
    """0.5 to 3 cells beyond each face of the box, at +-1e19 (finite squared distances near FLT_MAX), at +-1e30 (infinite ones)
    and at -0.0."""
    q, t, k, thr = outside_scene()
    lab = check_both(ctx, q, t, k, thr)
    assert 0 < lab.sum() < len(lab)
    assert lab[-14:-3].all()          # the huge queries are far


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 7, 16])
def test_knn_diff_with_awkward_setup(k):
    """40 ragged keyframes (some empty) against poses 5..44 of 50, a non-identity extrinsic and transform order 1."""
    import lt_mapper_b200 as ltr
    rng = np.random.default_rng(40 + k)
    sizes = rng.integers(0, 3000, 40)
    sizes[[0, 7, 8, 39]] = 0
    sizes[3] = 1
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    scans = xyzi(rng.normal(0, 6, (off[-1], 3)))
    poses = np.repeat(I4[None], 50, 0)
    for p in poses:
        a = rng.uniform(-np.pi, np.pi)
        p[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
        p[:3, 3] = rng.uniform(-10, 10, 3)
    inv = oracle.inverse_poses(poses)
    l2b = np.eye(4)
    b = 0.3
    l2b[:3, :3] = [[np.cos(b), 0, np.sin(b)], [0, 1, 0], [-np.sin(b), 0, np.cos(b)]]
    l2b[:3, 3] = [0.25, -0.1, 1.7]
    target = xyzi(rng.uniform(-16, 16, (60000, 3)) * [1, 1, 0.4], 10**6)
    thr = 0.05 * k
    with ltr.Context(lidar2base=l2b, base2lidar=oracle.inverse4x4(l2b), transform_order=1) as c:
        ss = c.scanset_upload(scans, off)
        ps = c.poses_upload(poses, inv)
        th = c.cloud_upload(target)
        co, di = c.knn_diff(ss, ps, th, k, thr, pose_offset=5)
        cp, coff = c.scanset_download(co)
        dp, doff = c.scanset_download(di)
    assert len(coff) == len(doff) == 41
    nd = 0
    for kf in range(40):
        s = scans[off[kf]:off[kf + 1]]
        lab, eco, edi = oracle.knn_partition(s, poses[5 + kf], inv[5 + kf], target, k, thr, lidar2base=l2b, order=1)
        assert np.array_equal(bits(cp[coff[kf]:coff[kf + 1]]), bits(eco)), kf
        assert np.array_equal(bits(dp[doff[kf]:doff[kf + 1]]), bits(edi)), kf
        nd += len(edi)
    assert 0 < nd < len(scans)


@pytest.mark.gpu
def test_benchmark_shape(ctx):
    """4M queries against 1M targets, k = 2, thr = 0.01 (the shape DESIGN quotes for the kNN kernel)."""
    rng = np.random.default_rng(4)
    t = rng.uniform(0, 1, (1_000_000, 3)) * [100, 100, 10]
    q = rng.uniform(0, 1, (4_000_000, 3)) * [100, 100, 10]
    q[:2_000_000] = t[rng.integers(0, len(t), 2_000_000)] + rng.normal(0, 0.05, (2_000_000, 3))
    q, t = xyzi(q), xyzi(t)
    lab = ref_labels(q, t, 2, 0.01)
    check_split(ctx, q, t, 2, 0.01, lab)
    assert 0.01 < lab.mean() < 0.99


NONFINITE_CHILD = textwrap.dedent("""
    import sys
    sys.path.insert(0, {root!r})
    import numpy as np
    import lt_mapper_b200 as ltr
    rng = np.random.default_rng(0)
    good = np.concatenate([rng.uniform(-5, 5, (5000, 3)), np.zeros((5000, 1))], 1).astype(np.float32)
    cases = {{}}
    for name, row, col, v in (("+inf", 17, 0, np.inf), ("-inf", 4000, 2, -np.inf), ("nan", 2500, 1, np.nan)):
        t = good.copy(); t[row, col] = v; cases[name] = t
    cases["all nan"] = np.full((300, 4), np.nan, np.float32)
    I4 = np.eye(4)[None]
    with ltr.Context() as ctx:
        q = ctx.cloud_upload(good[:1000])
        ss = ctx.scanset_upload(good[:1000], [0, 400, 1000])
        ps = ctx.poses_upload(np.repeat(I4, 2, 0), np.repeat(I4, 2, 0))
        targets = {{name: ctx.cloud_upload(t) for name, t in cases.items()}}
        base = ctx.memory_stats()[0]
        for name, th in targets.items():
            for entry, call in (("ltr_knn_split_cloud", lambda: ctx.knn_split_cloud(q, th, 2, 0.01)),
                                ("ltr_knn_diff", lambda: ctx.knn_diff(ss, ps, th, 2, 0.01)),
                                ("ltr_voxel_centroid", lambda: ctx.voxel_centroid(th, 0.1))):
                try:
                    call()
                except ltr.LtrError as e:
                    assert e.code == -3, (name, entry, e)
                else:
                    raise AssertionError(f"{{entry}} accepted a target with {{name}} coordinates")
                assert ctx.memory_stats()[0] == base, (name, entry)
    print("nonfinite ok")
""")


@pytest.mark.gpu
def test_non_finite_targets_are_rejected():
    """+inf, -inf, a NaN among finite points, all NaN: an error (not an endless cell-growth loop), with all scratch returned.  Runs in
    a child process so that a regression fails by timeout instead of hanging the suite."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", NONFINITE_CHILD.format(root=ROOT)]
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=120)
    except subprocess.TimeoutExpired:
        pytest.fail("the kNN calls on non-finite targets did not return within 120 s")
    assert r.returncode == 0 and "nonfinite ok" in r.stdout, r.stdout + r.stderr


# ---------------------------------------------------------------------------------------------------------------- CPU self-checks
@pytest.mark.parametrize("thr", THRS)
def test_selfcheck_density_scene_mixes_labels_for_every_k(thr):
    q, t = density_scene(thr)
    for k in range(1, 17):
        assert len(t) >= k and grid_geometry(t, k, thr)[2] == 0
        assert 0.1 < ref_labels(q, t, k, thr).mean() < 0.9, k


@pytest.mark.parametrize("k", [1, 2, 3, 5, 7, 16])
def test_selfcheck_threshold_sets(k):
    """Every hand-built set has exact squared distances at both offsets and gives its intended label."""
    for offset in (0.0, 3e5):
        centre = np.full(3, offset)
        for m, thr, expect, what in threshold_sets(k, seed=k):
            t = xyzi(axis_targets(centre, m))
            assert np.array_equal(t[:, :3].astype(np.float64), axis_targets(centre, m))      # exact in f32
            lab = ref_labels(xyzi(centre), t, k, float(thr))
            assert lab[0] == expect, what


@pytest.mark.parametrize("k,thr", [(1, 0.01), (1, 1.0), (4, 0.04), (16, 0.01), (16, 1.0)])
def test_selfcheck_reach_scene(k, thr):
    """The grid does not grow, half the queries are on faces (0..2 ulps off), the far neighbours straddle k*thr, and some near
    points have their last neighbour more than 0.999 * sqrt(k*thr) across a face."""
    q, t, cell = reach_scene(k, thr, seed=k)
    c2, origin, steps = grid_geometry(t, k, thr)
    assert steps == 0 and c2 == cell
    rel = (q[:, :3].astype(np.float64) - origin) / cell
    assert (np.abs(rel - np.round(rel)) < 1e-3).all(1).mean() > 0.45
    lab = ref_labels(q, t, k, thr)
    assert 0.2 < lab.mean() < 0.8
    # near points whose last neighbour is two cells away in a grid whose cells are only 0.999 * sqrt(k*thr): what the 1.001 slack is for
    short = math.sqrt(k * float(F32(thr))) * 0.999 + 1e-6
    far_pt = t[len(q) * (k - 1):len(q) * k, :3].astype(np.float64)
    cq = np.floor((q[:, :3] - (1.0 - short)) / short)
    ct = np.floor((far_pt - (1.0 - short)) / short)
    assert ((np.abs(cq - ct) >= 2).any(1) & (lab == 0)).sum() >= 5


def test_selfcheck_growth_scene_grows_the_cells():
    q, t = growth_scene()
    cell, _, steps = grid_geometry(t, 1, 1e-4)
    assert steps > 20 and cell > 100 * 0.01


def test_selfcheck_outside_scene():
    q, t, k, thr = outside_scene()
    cell, origin, _ = grid_geometry(t, k, thr)
    lo, hi = t[:, :3].min(0), t[:, :3].max(0)
    assert ((q[:, :3] < lo) | (q[:, :3] > hi)).any(1).all()
    d = oracle.knn_dists(q[-14:-3], t, k)
    assert np.isfinite(d[:6]).all() and np.isinf(d[6:]).all()        # +-1e19: finite squared distances; +-1e30: infinite
