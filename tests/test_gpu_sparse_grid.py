"""The exact nearest-neighbour searches over the sparse grid levels of sparse_grid.cuh (scan-side removal's k-NN averages, scanside.cu;
ICP's nearest neighbour with the lowest index on ties, icp.cu) at the shapes and edges the pipeline never reaches.

ltr_debug_exact_knn_avg and ltr_debug_nearest run the production search on any query set, so every value is compared query by query,
bit for bit: the average with a brute force in this module (FLANN's L2_Simple op by op in f32, the k smallest sorted, summed ascending in
f64, (float)sum / (float)k), and the nearest neighbour with the minimum distance and the lowest index at it.  Where brute force is too
slow the references are oracle.knn_dists and _icp_oracle.Target.nn, spot-checked against brute force.  The end-to-end tests run
ltr_scanside_split and ltr_icp_refine + ltr_knn_diff_refined at the same shapes against their CPU restatements.

Covered: every k on a scene whose queries settle on each level; queries on cell faces and corners; the k-th neighbour in each of the 26
directions around the shell radii; a neighbour across a face closer than the shell-0 bound; lattices on the cell faces of two levels with
ties at the k-th distance and at the nearest one; targets of fewer than k points; queries outside the box, up to infinite distances;
corridors that scale the finest cell and build all eight levels; ragged and identical keyframes, and 8192 of them in one launch; the
pipeline's shape.  The tests without the gpu mark check on the CPU, with a Python copy of the level geometry and the shell stop rule,
that each scene takes the path its GPU test claims.
"""
import functools
import math

import numpy as np
import pytest

import oracle
import _icp_oracle as io
import _scanside_oracle as so

F32 = np.float32
I4 = np.eye(4)

# sparse_grid.cuh / scanside.cu / icp.cu
CELL_BITS = 17
SEG_SHIFT = 3 * CELL_BITS
MAX_SEGMENTS = 1 << (64 - SEG_SHIFT)
MAX_DIM = (1 << CELL_BITS) - 1
CELL0 = 0.25
MAX_LEVELS = 8
FINAL_DIM = 10
BOUNDED_SHELLS = 2


# ---------------------------------------------------------------------------------------------------------------- geometry model
def pyramid_cell0(mn, mx):
    """Pyramid::init: the finest cell side, scaled up so that the finest level's indices stay below 2^17."""
    ext = max(float(mx[d]) - float(mn[d]) for d in range(3))
    return max(CELL0, ext / (MAX_DIM - 4))


def level(mn, mx, m, cell0=None):
    """Pyramid::get + build_level for level m of the box [mn, mx] (float32 per axis)."""
    cell0 = pyramid_cell0(mn, mx) if cell0 is None else cell0
    cell = cell0 * 4.0 ** m
    dmax = max(math.floor((float(mx[d]) - float(mn[d])) / cell) + 3 for d in range(3))
    inv = 1.0 / cell
    origin = np.array([float(mn[d]) - cell for d in range(3)])
    dim = np.array([math.floor((float(mx[d]) - origin[d]) * inv) + 2 for d in range(3)], np.int64)
    return dict(cell=1.0 / inv, inv=inv, origin=origin, dim=dim, natural=dmax <= FINAL_DIM, final=dmax <= FINAL_DIM or m == MAX_LEVELS - 1)


def levels(mn, mx):
    """Every level Pyramid::get can build for the box, finest first, up to the final one."""
    out = []
    for m in range(MAX_LEVELS):
        out.append(level(mn, mx, m))
        if out[-1]["final"]:
            return out
    raise AssertionError("no final level")


def cell_index(v, L):
    """cell_index: floor(fl(fl(v - origin) * inv_cell)) in double, clamped to +-2^40."""
    t = (np.asarray(v, np.float64) - L["origin"]) * L["inv"]
    return np.floor(np.clip(t, -2.0 ** 40, 2.0 ** 40)).astype(np.int64)


def shell_bound(s, cell):
    r = (s - 2.0 ** -6) * cell
    return r * r * (1.0 - 2.0 ** -20)


def box(t):
    t = np.asarray(t, F32)[:, :3]
    return t.min(0), t.max(0)


def settle_levels(q, t, k, nearest=False, chunk=64):
    """The level on which each query of q is answered (shell_search with Best<k>, or Nearest when `nearest`), one segment."""
    q, t = np.asarray(q, F32)[:, :3], np.asarray(t, F32)[:, :3]
    mn, mx = box(t)
    lv = levels(mn, mx)
    out = np.full(len(q), len(lv) - 1)
    cts = [np.minimum(np.maximum(cell_index(t, L), 0), L["dim"] - 1) for L in lv]
    for a in range(0, len(q), chunk):
        qq = q[a:a + chunk]
        D = l2(qq, t)
        todo = np.ones(len(qq), bool)
        for li, L in enumerate(lv[:-1]):
            cq = cell_index(qq, L)
            hi = L["dim"] - 1
            s0 = np.maximum(np.maximum(-cq, cq - hi).max(1), 0)
            cover = np.maximum(np.maximum(cq, hi - cq).max(1), 0)
            cheb = np.abs(cts[li][None, :, :] - cq[:, None, :]).max(2)
            done = np.zeros(len(qq), bool)
            for s in range(BOUNDED_SHELLS + 1):
                live = todo & ~done & (s0 <= s)
                if not live.any():
                    continue
                blk = cheb <= s
                cnt = blk.sum(1)
                need = 1 if nearest else k
                Dm = np.where(blk, D, np.inf)
                dk = np.partition(Dm, need - 1, axis=1)[:, need - 1].astype(np.float64) if len(t) >= need else np.full(len(qq), np.inf)
                ok = (cnt >= need) & (s > 0) & (dk <= shell_bound(s, L["cell"]))
                if not nearest:
                    ok |= (cnt >= need) & (dk == 0.0)
                ok |= s >= cover
                done |= live & ok
            out[a:a + chunk][todo & done] = li
            todo &= ~done
    return out


# ---------------------------------------------------------------------------------------------------------------- references
def l2(q, t):
    """FLANN L2_Simple in f32, op by op: ((dx*dx) + dy*dy) + dz*dz, dx = query - point; (len(q), len(t))."""
    d = np.asarray(q, F32)[:, None, :3] - np.asarray(t, F32)[None, :, :3]
    with np.errstate(over="ignore"):
        return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def brute_smallest(q, t, kmax=16, budget=4_000_000):
    """The kmax smallest L2_Simple values per query, ascending, +inf past the target's size."""
    out = np.full((len(q), kmax), np.inf, F32)
    m = min(kmax, len(t))
    step = max(1, budget // max(len(t), 1))
    for a in range(0, len(q), step):
        D = l2(q[a:a + step], t)
        if m < len(t):
            D = np.partition(D, m - 1, axis=1)[:, :m]
        out[a:a + step, :m] = np.sort(D, axis=1)[:, :m]
    return out


def avg_of(dk, k, n_target):
    """(float)(sum in double, ascending, of the min(k, n) smallest) / (float)k."""
    s = np.zeros(len(dk))
    for j in range(min(k, n_target)):
        s = s + dk[:, j].astype(np.float64)
    with np.errstate(over="ignore"):
        return s.astype(F32) / F32(k)


def brute_nearest(q, t, budget=4_000_000):
    """(smallest L2_Simple value, lowest target index at it) per query."""
    d = np.empty(len(q), F32)
    idx = np.empty(len(q), np.int64)
    step = max(1, budget // max(len(t), 1))
    for a in range(0, len(q), step):
        D = l2(q[a:a + step], t)
        d[a:a + step] = D.min(1)
        idx[a:a + step] = D.argmin(1)             # the first index at the minimum
    return d, idx


def kd_smallest(q, t, k, spot=20_000_000):
    """oracle.knn_dists, spot-checked against brute force on as many queries as `spot` distance evaluations allow."""
    d = oracle.knn_dists(xyzi(q), xyzi(t), k)
    m = max(1, min(len(q), spot // max(len(t), 1)))
    sel = np.linspace(0, len(q) - 1, m).astype(np.int64)
    assert np.array_equal(bits(d[sel]), bits(brute_smallest(q[sel], t, k)))
    return d


def kd_nearest(q, t, spot=20_000_000):
    """_icp_oracle.Target.nn, spot-checked against brute force."""
    d, idx = io.Target(xyzi(t)).nn(xyzi(q))
    m = max(1, min(len(q), spot // max(len(t), 1)))
    sel = np.linspace(0, len(q) - 1, m).astype(np.int64)
    bd, bi = brute_nearest(q[sel], t)
    fin = np.isfinite(bd)
    assert np.array_equal(bits(d[sel]), bits(bd)) and np.array_equal(idx[sel][fin], bi[fin])
    return d, idx


def xyzi(p):
    p = np.asarray(p, F32)
    if p.shape[1] == 4:
        return p
    return np.concatenate([p, np.zeros((len(p), 1), F32)], 1)


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def f32(a):
    return np.asarray(a, np.float64).astype(F32)


# ---------------------------------------------------------------------------------------------------------------- scenes
def slab_scene(seed=0):
    """Four slabs along x of decreasing density (100, 2, 0.03 and 0.008 points per m^3) in an 8 m x 8 m section, 504 m long: for every
    k some queries settle on level 0 (0.25 m cells), some on 1, 2 and 3, and queries 60-200 m above the slabs on the final level 4."""
    rng = np.random.default_rng(seed)
    parts, qs, x0 = [], [], 0.0
    for rho, length in ((100, 4.0), (2, 20.0), (0.03, 80.0), (0.008, 400.0)):
        n = int(rho * 64 * length)
        p = rng.uniform(0, 1, (n, 3)) * [length, 8, 8] + [x0, 0, 0]
        parts.append(p)
        qs.append(rng.uniform(0, 1, (1200, 3)) * [length, 8, 8] + [x0, 0, 0])
        qs.append(p[rng.integers(0, n, 400)] + rng.normal(0, 0.05, (400, 3)))
        x0 += length
    above = rng.uniform(0, 1, (200, 3)) * [x0, 8, 8]
    above[:, 2] += rng.choice([60.0, 200.0], 200)
    qs.append(above)
    return f32(np.concatenate(qs)), f32(np.concatenate(parts))


def face_scene(seed=1):
    """Queries on the cell faces, edges and corners of level 0 (0.25 m) and level 1 (1 m), 0..2 ulps off, against a 20 m box (exact
    corners 0 and 20, so the level origins are -0.25 and -1) with a dense 5 m corner and a sparse rest."""
    rng = np.random.default_rng(seed)
    t = np.concatenate([rng.uniform(0, 5, (12000, 3)), rng.uniform(0, 20, (6000, 3)), [[0, 0, 0], [20, 20, 20]]])
    q = []
    for cell in (0.25, 1.0):
        n = 3000
        p = rng.uniform(0.5, 19.5, (n, 3))
        p[: n // 2] = rng.uniform(0.25, 4.75, (n // 2, 3))
        on = rng.random((n, 3)) < 0.6
        on[np.arange(n), rng.integers(0, 3, n)] = True               # at least one axis on a face
        p = np.where(on, np.round(p / cell) * cell, p)
        p = f32(p)
        nudge = np.where(on, rng.integers(-2, 3, (n, 3)), 0)
        towards = np.where(nudge > 0, F32(np.inf), F32(-np.inf))
        for step in (1, 2):
            p = np.where(np.abs(nudge) >= step, np.nextafter(p, towards), p)
        q.append(p)
    return np.concatenate(q), f32(t)


DIRS = np.array([(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1) if (a, b, c) != (0, 0, 0)], np.float64)


def direction_scene(k, seed=2, cell=0.25):
    """Isolated queries 6 m apart; k - 1 targets on each query and two more, in two of the 26 directions, at distances straddling s*c
    and the shell radius (s - 2^-6) c (s = 1, 2, 3; s = 3 is past the bounded shells of level 0) by up to a few parts in 1e6."""
    rng = np.random.default_rng(seed + k)
    qs, ts = [], []
    g = 0
    for s in (1, 2, 3):
        for base in (s * cell, (s - 2.0 ** -6) * cell):
            for di in range(26):
                for rep in range(3):
                    centre = np.array([g % 20, (g // 20) % 20, g // 400], np.float64) * 6.0 + 2.0
                    g += 1
                    qq = f32(centre + rng.uniform(0, cell, 3) * (rep > 0))        # rep 0: on a corner of a level-0 cell
                    r1 = base * (1 + rng.choice([-2e-6, -3e-7, 0.0, 3e-7, 2e-6]))
                    r2 = base * (1 + rng.choice([-2e-6, -3e-7, 0.0, 3e-7, 2e-6]))
                    d2 = DIRS[rng.integers(0, 26)]
                    p1 = qq + DIRS[di] / np.linalg.norm(DIRS[di]) * r1
                    p2 = qq + d2 / np.linalg.norm(d2) * r2
                    qs.append(qq)
                    ts.extend([qq] * (k - 1) + [p1, p2])
    ts.append(np.zeros(3))                                  # the box minimum: level-0 faces at multiples of c
    return f32(qs), f32(ts)


ANCHOR = np.zeros((1, 3), F32)      # the box minimum of the across-face scene: level-0 faces at multiples of 0.25


def across_face_scene(seed=3, cell=0.25):
    """A query just inside a level-0 cell face, a target inside its own cell at d_in < c/64 and one just across the face at
    d_out < d_in, across each of the six faces; the k - 1 nearest are copies of the query for k > 1.  Stopping in shell 0 on
    D_k <= ((0 - 2^-6) c)^2 would take d_in."""
    rng = np.random.default_rng(seed)
    qs, inner, outer = [], [], []
    for g in range(600):
        centre = np.array([g % 10, (g // 10) % 10, g // 100], np.float64) * 4.0 + 1.0     # multiples of 0.25: cell faces
        ax, sgn = g % 3, (1 if (g // 3) % 2 else -1)
        a = rng.uniform(2e-4, 1e-3)                     # query this far inside the face
        d_in = rng.uniform(2.5e-3, 3.8e-3)               # < c/64 = 3.9e-3
        d_out = rng.uniform(a + 1e-4, d_in - 2e-4)
        e = np.zeros(3); e[ax] = sgn
        q = centre - e * a + rng.uniform(0.05, 0.2, 3) * (1 - np.abs(e)) * cell
        qs.append(q)
        inner.append(q - e * d_in)
        outer.append(q + e * d_out)
    return f32(qs), f32(inner), f32(outer)


def lattice_scene(spacing, seed=4, side=10):
    """A lattice of `spacing` starting at 3.0 (on the cell faces of level 0 and, for spacing 1, of level 1), stored twice: once in
    reversed index order, then forwards.  Queries: lattice points (ties at 0 between the copies), midpoints along 1, 2 and 3 axes (ties
    between 2, 4 and 8 points in different cells, the lowest index in the cell searched last) and jittered points."""
    rng = np.random.default_rng(seed)
    ax = 3.0 + np.arange(side) * spacing
    L = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    t = np.concatenate([L[::-1], L])
    base = L[rng.integers(0, len(L), 1500)]
    mids = []
    for naxes in (1, 2, 3):
        off = np.zeros((500, 3))
        for r in range(500):
            off[r, rng.permutation(3)[:naxes]] = 0.5 * spacing
        mids.append(base[:500] + off)
    q = np.concatenate([base[:400]] + mids + [base[:400] + rng.normal(0, 0.3 * spacing, (400, 3))])
    return f32(q), f32(t)


def small_target_scene(n, seed=5):
    """n target points over a 50 m box (levels 0-2 bounded, 3 final); queries around it and on the points."""
    rng = np.random.default_rng(seed + n)
    t = rng.uniform(0, 50, (n, 3))
    if n >= 2:
        t[0], t[1] = [0, 0, 0], [50, 50, 50]
    q = np.concatenate([rng.uniform(-10, 60, (1500, 3)), t[rng.integers(0, n, 300)] + rng.normal(0, 0.2, (300, 3))])
    return f32(q), f32(t)


def outside_scene(seed=6):
    """A 30 m box; queries 0.5 to 3 cells (of levels 0 and 1) beyond each face, at +-1e19 (finite squared distances near FLT_MAX), at
    +-1e30 (infinite ones) and at -0.0."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(0, 30, (6000, 3))
    t[0], t[1] = [0, 0, 0], [30, 30, 30]
    q = []
    for cell in (0.25, 1.0):
        for d in range(3):
            for s in (-1, 1):
                for f in np.arange(0.5, 3.01, 0.25):
                    p = rng.uniform(0, 30, (25, 3))
                    p[:, d] = (30 + f * cell) if s > 0 else -f * cell
                    q.append(p)
    special = [[1e19, 5, 5], [-1e19, 5, 5], [5, 1e19, 5], [5, 5, -1e19], [1e19, 1e19, 1e19], [-1e19, 1e19, -1e19],
               [1e30, 5, 5], [-1e30, 5, 5], [5, -1e30, 5], [5, 5, 1e30], [1e30, -1e30, 1e30],
               [-0.0, -0.0, -0.0], [-0.0, 5, 5], [5, -0.0, 0.0]]
    return np.concatenate([f32(np.concatenate(q)), np.array(special, F32)]), f32(t)


def corridor_scene(length, seed=7):
    """A corridor `length` m x 20 m x 5 m: 200 blocks of 300 points along the first half, pairs of points 8 km apart along the second
    half (fewer than k = 4 points for 8 km: those queries settle only on the final level), queries on and between them."""
    rng = np.random.default_rng(seed)
    blocks = [rng.uniform(0, 1, (300, 3)) * [10, 20, 5] + [i * length / 400, 0, 0] for i in range(200)]
    xs = np.arange(length / 2 + 1000, length - 500, 8000)
    pairs = [np.array([[x, 10, 2], [x + 1, 10, 2.5]]) for x in xs]
    t = np.concatenate(blocks + pairs + [np.array([[0, 0, 0], [length, 20, 5]])])
    b = np.concatenate(blocks)
    q = np.concatenate([b[rng.integers(0, len(b), 20000)] + rng.normal(0, 0.3, (20000, 3)),
                        rng.uniform(0, 1, (4000, 3)) * [length, 20, 5],
                        np.concatenate([p[0] + rng.normal(0, 3, (60, 3)) for p in pairs])])
    return f32(q), f32(t)


def ragged_keyframes(seed=8):
    """Keyframes of 0 .. 400 points (some empty, some below k), three of them exact copies of another."""
    rng = np.random.default_rng(seed)
    sizes = [0, 1, 2, 5, 15, 16, 17, 400, 0, 3, 250, 60]
    kfs = [rng.normal(0, 1.5, (n, 3)) + rng.uniform(-3, 3, 3) for n in sizes]
    kfs += [kfs[7], kfs[10], kfs[4]]
    return [f32(k) for k in kfs]


def many_keyframes(K=MAX_SEGMENTS, seed=9):
    """K keyframes of 0..20 points, each the first points of one common pattern: every keyframe has copies in all the others."""
    rng = np.random.default_rng(seed)
    pattern = f32(rng.normal(0, 0.6, (20, 3)))
    sizes = rng.integers(0, 21, K)
    sizes[[0, K - 1]] = 20
    return pattern, sizes


def offsets_of(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------- GPU helpers
@pytest.fixture(scope="module")
def ctx():
    import lt_mapper_b200 as ltr
    c = ltr.Context()
    yield c
    c.close()


def dev_avg(ctx, q, ks, t=None, offsets=None):
    """{k: (avg, unsettled)} of ltr_debug_exact_knn_avg: one keyframe of queries against t, or every keyframe of q against itself."""
    qs = ctx.scanset_upload(xyzi(q), [0, len(q)] if offsets is None else offsets)
    th = None if t is None else ctx.cloud_upload(xyzi(t))
    out = {k: ctx.debug_exact_knn_avg(qs, k, th) for k in ks}
    ctx.scanset_free(qs)
    if th is not None:
        ctx.cloud_free(th)
    return out


def dev_nearest(ctx, q, t):
    qh, th = ctx.cloud_upload(xyzi(q)), ctx.cloud_upload(xyzi(t))
    d, idx = ctx.debug_nearest(qh, th)
    ctx.cloud_free(qh)
    ctx.cloud_free(th)
    return d, idx


def assert_avg(got, dk, k, n_target, what=""):
    exp = avg_of(dk, k, n_target)
    bad = np.nonzero(bits(got) != bits(exp))[0]
    assert len(bad) == 0, f"{what} k={k}: {len(bad)} queries differ, first {bad[:5]}: {got[bad[:5]]} vs {exp[bad[:5]]}"


def assert_nearest(got, exp):
    d, idx = got
    ed, ei = exp
    assert np.array_equal(bits(d), bits(ed)), np.nonzero(bits(d) != bits(ed))[0][:10]
    fin = np.isfinite(ed)
    bad = np.nonzero(fin & (idx != ei))[0]
    assert len(bad) == 0, f"{len(bad)} indices differ, first {bad[:5]}: {idx[bad[:5]]} vs {ei[bad[:5]]}"


def check_scene(ctx, q, t, ks, nearest=True, brute=True):
    dk = brute_smallest(q, t, max(ks)) if brute else kd_smallest(q, t, max(ks))
    out = dev_avg(ctx, q, ks, t)
    for k in ks:
        assert_avg(out[k][0], dk, k, len(t))
    if nearest:
        assert_nearest(dev_nearest(ctx, q, t), brute_nearest(q, t) if brute else kd_nearest(q, t))
    return out


@functools.lru_cache(maxsize=None)
def slab_reference():
    q, t = slab_scene()
    return q, t, brute_smallest(q, t, 16)


# ---------------------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
def test_every_k_on_the_density_slabs(ctx):
    q, t, dk = slab_reference()
    out = dev_avg(ctx, q, range(1, 17), t)
    for k in range(1, 17):
        avg, unsettled = out[k]
        assert_avg(avg, dk, k, len(t), "slabs")
        assert 0 < unsettled < len(q), k
    assert_nearest(dev_nearest(ctx, q, t), brute_nearest(q, t))


@pytest.mark.gpu
def test_queries_on_cell_faces_and_corners(ctx):
    q, t = face_scene()
    check_scene(ctx, q, t, (1, 2, 4, 9, 16))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 16])
def test_kth_neighbour_in_every_direction_around_the_shell_radii(ctx, k):
    q, t = direction_scene(k)
    check_scene(ctx, q, t, (k,), nearest=k == 1)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 5, 16])
def test_neighbour_across_a_face_closer_than_the_shell_zero_bound(ctx, k):
    q, inner, outer = across_face_scene()
    t = np.concatenate([np.repeat(q, k - 1, 0), inner, outer, ANCHOR])
    dk = brute_smallest(q, t, k)
    assert_avg(dev_avg(ctx, q, (k,), t)[k][0], dk, k, len(t), "across a face")
    if k == 1:
        assert_nearest(dev_nearest(ctx, q, t), brute_nearest(q, t))


@pytest.mark.gpu
@pytest.mark.parametrize("spacing", [0.25, 1.0])
def test_lattices_on_cell_faces_with_ties(ctx, spacing):
    q, t = lattice_scene(spacing)
    check_scene(ctx, q, t, (1, 2, 3, 4, 7, 8, 9, 16))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 5, 16])
def test_targets_of_fewer_than_k_points_and_of_k(ctx, k):
    for n in range(1, k + 1):
        q, t = small_target_scene(n)
        out = check_scene(ctx, q, t, (k,), nearest=n <= 2 or n == k)
        if n < k and n >= 2:
            assert out[k][1] == len(q), (n, out[k][1])      # nothing settles on the bounded levels


@pytest.mark.gpu
def test_queries_outside_the_box(ctx):
    q, t = outside_scene()
    out = check_scene(ctx, q, t, (1, 2, 16))
    assert np.isinf(out[2][0][-8:-3]).all() and np.isfinite(out[1][0][-14:-8]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("length", [40000.0, 30000.0])
def test_corridor_builds_every_level(ctx, length):
    q, t = corridor_scene(length)
    out = check_scene(ctx, q, t, (1, 4, 16), brute=False)
    assert out[4][1] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 2, 4, 16])
def test_self_mode_ragged_and_identical_keyframes(ctx, k):
    kfs = ragged_keyframes()
    off = offsets_of([len(x) for x in kfs])
    q = np.concatenate(kfs)
    avg, _ = dev_avg(ctx, q, (k,), offsets=off)[k]
    for j, p in enumerate(kfs):
        if len(p):
            assert_avg(avg[off[j]:off[j + 1]], brute_smallest(p, p, k), k, len(p), f"keyframe {j}")


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 4])
def test_self_mode_8192_keyframes_in_one_launch(ctx, k):
    pattern, sizes = many_keyframes()
    off = offsets_of(sizes)
    q = np.concatenate([pattern[:n] for n in sizes])
    avg, _ = dev_avg(ctx, q, (k,), offsets=off)[k]
    exp = {n: avg_of(brute_smallest(pattern[:n], pattern[:n], k), k, n) for n in range(1, 21)}
    for j, n in enumerate(sizes):
        if n:
            assert np.array_equal(bits(avg[off[j]:off[j + 1]]), bits(exp[n])), (j, n)


@pytest.mark.gpu
def test_debug_entry_points_reject_bad_input(ctx):
    import lt_mapper_b200 as ltr
    qs = ctx.scanset_upload(xyzi(np.zeros((MAX_SEGMENTS + 1, 3), F32)), np.arange(MAX_SEGMENTS + 2))
    th = ctx.cloud_upload(xyzi(np.zeros((1, 3), F32)))
    with pytest.raises(ltr.LtrError):
        ctx.debug_exact_knn_avg(qs, 2)
    ctx.debug_exact_knn_avg(qs, 2, th)                          # against a target: one segment, accepted
    for k in (0, 17):
        with pytest.raises(ltr.LtrError):
            ctx.debug_exact_knn_avg(qs, k, th)
    empty = ctx.cloud_upload(np.zeros((0, 4), F32))
    bad = ctx.cloud_upload(np.array([[0, 0, 0, 0], [np.inf, 0, 0, 0]], F32))
    for h in (empty, bad):
        with pytest.raises(ltr.LtrError):
            ctx.debug_exact_knn_avg(qs, 2, h)
        with pytest.raises(ltr.LtrError):
            ctx.debug_nearest(th, h)
    with pytest.raises(ltr.LtrError):
        ctx.debug_nearest(bad, th)
    for h in (th, empty, bad):
        ctx.cloud_free(h)
    ctx.scanset_free(qs)


def pipeline_clouds(ctx):
    """Global scans of 40 keyframes of configs[2]'s scan shape (64 x 1800) as queries (4.1 M points), the other session's 0.05 m map
    (1.8 M points) as target."""
    import synth
    c, qsess = synth.make_pair(40, beams=64, az_steps=1800)
    inv = oracle.inverse_poses(qsess.poses)
    ss = ctx.scanset_upload(qsess.xyzi, qsess.offsets)
    ps = ctx.poses_upload(qsess.poses, inv)
    raw = ctx.merge_scans_global(ss, ps)
    mh = ctx.voxel_centroid(raw, 0.05)
    m = ctx.cloud_download(mh).copy()
    cs = ctx.scanset_upload(c.xyzi, c.offsets)
    cp = ctx.poses_upload(c.poses, oracle.inverse_poses(c.poses))
    gh = ctx.merge_scans_global(cs, cp)
    g = ctx.cloud_download(gh).copy()
    for h in (raw, mh, gh):
        ctx.cloud_free(h)
    for h in (ss, cs):
        ctx.scanset_free(h)
    for h in (ps, cp):
        ctx.poses_free(h)
    return g, c.offsets, m


@pytest.mark.gpu
def test_pipeline_shape(ctx):
    g, off, m = pipeline_clouds(ctx)
    assert len(g) == off[-1] > 4_000_000 and len(m) > 1_500_000
    q = g[:, :3]
    out = dev_avg(ctx, q, (2,), m[:, :3])
    assert_avg(out[2][0], kd_smallest(q, m[:, :3], 2), 2, len(m), "map")
    avg, _ = dev_avg(ctx, q, (2,), offsets=off)[2]
    for j in range(len(off) - 1):
        p = q[off[j]:off[j + 1]]
        assert_avg(avg[off[j]:off[j + 1]], oracle.knn_dists(xyzi(p), xyzi(p), 2), 2, len(p), f"keyframe {j}")


# ---- end to end through the public entry points
def _scanside_device(ctx, xyz, off, poses, mp, criterion, k, thr):
    ss = ctx.scanset_upload(xyzi(xyz), off)
    ps = ctx.poses_upload(poses, oracle.inverse_poses(poses))
    mh = ctx.cloud_upload(xyzi(mp))
    st, dy = ctx.scanside_split(ss, ps, mh, criterion, k, thr)
    stats = ctx.scanside_stats()
    out = []
    for h in (st, dy):
        pts, o = ctx.scanset_download(h)
        out.append([pts[o[j]:o[j + 1]] for j in range(len(o) - 1)])
        ctx.scanset_free(h)
    ctx.scanset_free(ss)
    ctx.poses_free(ps)
    ctx.cloud_free(mh)
    return out, stats


def _assert_split(dev, xyz, off, poses, mp, criterion, k, thr):
    exp = so.split_session(xyzi(xyz), off, poses, oracle.inverse_poses(poses), xyzi(mp), criterion, k, thr)
    for part in range(2):
        for j, (a, b) in enumerate(zip(dev[part], exp[part])):
            assert a.shape == b.shape and np.array_equal(bits(a), bits(b)), (part, j)


@pytest.mark.gpu
@pytest.mark.parametrize("criterion", [so.MAP, so.SCAN_MINUS_MAP])
def test_scanside_split_on_8200_keyframes(ctx, criterion):
    """Two launches, 8192 keyframes and 8: small copies of one pattern, moved by poses 0.5 m apart."""
    pattern, sizes = many_keyframes(8200)
    off = offsets_of(sizes)
    xyz = np.concatenate([pattern[:n] for n in sizes])
    poses = np.repeat(I4[None], 8200, 0)
    poses[:, 0, 3] = (np.arange(8200) % 100) * 0.5
    poses[:, 1, 3] = (np.arange(8200) // 100) * 0.5
    rng = np.random.default_rng(10)
    mp = f32(rng.uniform(0, 1, (2000, 3)) * [50, 41, 1] + [-1, -1, -0.5])
    dev, stats = _scanside_device(ctx, xyz, off, poses, mp, criterion, 3, 0.3)
    assert stats[3] == 2
    _assert_split(dev, xyz, off, poses, mp, criterion, 3, 0.3)


@pytest.mark.gpu
def test_scanside_split_on_a_corridor_session(ctx):
    """Six keyframes, each a slice of the 40 km corridor in its own frame, against the corridor: both expanding passes are used."""
    q, t = corridor_scene(40000.0)
    rng = np.random.default_rng(11)
    kfs, poses = [], []
    for j in range(6):
        p = q[rng.choice(len(q), 3000, replace=False)]
        T = I4.copy()
        T[:3, 3] = [j * 10.0, 0.5, 0.0]
        kfs.append(f32(p - T[:3, 3]))
        poses.append(T)
    xyz, off, poses = np.concatenate(kfs), offsets_of([len(x) for x in kfs]), np.stack(poses)
    dev, stats = _scanside_device(ctx, xyz, off, poses, t, so.SCAN_MINUS_MAP, 4, 0.2)
    assert stats[1] > 0 and stats[2] > 0, stats
    _assert_split(dev, xyz, off, poses, t, so.SCAN_MINUS_MAP, 4, 0.2)


@pytest.mark.gpu
def test_icp_against_a_corridor_target(ctx):
    """ltr_icp_refine + ltr_knn_diff_refined against the 40 km corridor: two keyframes on it with a pose error, one whose source lies
    100-150 m beside it (its correspondences come from level 4 or deeper), one in the sparse half."""
    from test_gpu_icp import _run
    q, t = corridor_scene(40000.0)
    rng = np.random.default_rng(12)
    blk = t[:3000]
    side = blk + [0, 120.0, 0]
    side[:, 1] += rng.uniform(0, 25, len(side))
    sparse = t[60000:60004] + rng.normal(0, 0.5, (4, 3))
    kfs = [f32(blk[:1500]), f32(blk[1500:]), f32(side), f32(sparse)]
    E = I4.copy()
    E[:3, 3] = [0.3, -0.2, 0.1]
    poses = np.stack([E, E, I4, I4])
    off = offsets_of([len(x) for x in kfs])
    _run(ctx, xyzi(np.concatenate(kfs)), off, poses, xyzi(t), xyzi(t), k=2, thr=0.05)


# ---------------------------------------------------------------------------------------------------------------- CPU self-checks
def test_selfcheck_last_level_is_always_naturally_final():
    """Over extents from 1 m to 1e7 m the coarsest level Pyramid::get builds has at most 10 cells per axis by itself: the
    `m == kGridMaxLevels - 1` term never decides."""
    for ext in np.geomspace(1.0, 1e7, 4000):
        mx = np.array([ext, ext / 3, 1.0], F32)
        lv = levels(np.zeros(3, F32), mx)
        assert lv[-1]["natural"], ext
        assert (lv[0]["dim"] < 2 ** CELL_BITS).all(), ext


def test_selfcheck_slab_scene_reaches_every_level():
    q, t, dk = slab_reference()
    lv = levels(*box(t))
    assert len(lv) == 5 and lv[0]["cell"] == 0.25
    sub = np.arange(0, len(q), 10)
    for k in (1, 4, 16):
        reached = set(settle_levels(q[sub], t, k).tolist())
        assert {0, 1, 2, 4} <= reached and (k == 1 or 3 in reached), (k, reached)
    assert set(settle_levels(q[sub], t, 1, nearest=True).tolist()) >= {0, 1, 2, 4}


def test_selfcheck_face_scene():
    q, t = face_scene()
    L0, L1 = level(*box(t), 0), level(*box(t), 1)
    assert L0["origin"][0] == -0.25 and L1["origin"][0] == -1.0
    for L, half in ((L0, slice(0, 3000)), (L1, slice(3000, 6000))):
        rel = (q[half].astype(np.float64) - L["origin"]) * L["inv"]
        near = np.abs(rel - np.round(rel)) < 1e-4
        assert near.any(1).all() and (near.sum(1) == 3).sum() > 50
        exact = rel == np.round(rel)
        assert exact.any(1).sum() > 300 and (near & ~exact).any(1).sum() > 300
    lv = settle_levels(q[::4], t, 4)
    assert {0, 1} <= set(lv.tolist())


def test_selfcheck_direction_scene():
    for k in (1, 3, 16):
        q, t = direction_scene(k)
        lv = settle_levels(q[::3], t, k)
        assert {0, 1} <= set(lv.tolist())
        dk = brute_smallest(q, t, k)[:, k - 1].astype(np.float64)
        for s in (1, 2, 3):
            r2 = (s * 0.25) ** 2
            assert ((dk > r2) & (dk < r2 * (1 + 1e-5))).any() and ((dk < r2) & (dk > r2 * (1 - 1e-5))).any(), (k, s)


def test_selfcheck_across_face_scene_needs_the_next_shell():
    q, inner, outer = across_face_scene()
    L = level(*box(np.concatenate([q, inner, outer, ANCHOR])), 0)
    c = L["cell"]
    assert c == 0.25
    cq, ci, co = cell_index(q, L), cell_index(inner, L), cell_index(outer, L)
    assert (cq == ci).all() and (np.abs(cq - co).max(1) == 1).all()
    d_in, d_out = l2(q, inner).diagonal(), l2(q, outer).diagonal()
    assert (d_out < d_in).all() and (d_in.astype(np.float64) <= shell_bound(0, c)).all()


def test_selfcheck_lattices_tie_across_cells_and_levels():
    for spacing in (0.25, 1.0):
        q, t = lattice_scene(spacing)
        L0 = level(*box(t), 0)
        rel = (t.astype(np.float64) - L0["origin"]) * L0["inv"]
        assert (rel == np.round(rel)).all()
        d, idx = brute_nearest(q, t)
        D = l2(q, t)
        ties = (D == d[:, None]).sum(1)
        assert (ties >= 2).all() and (ties >= 8).sum() > 100
        cells = cell_index(t, L0)
        first_in_key_order = np.array([np.nonzero(D[i] == d[i])[0][np.lexsort(cells[D[i] == d[i]].T)[0]] for i in range(len(q))])
        assert (first_in_key_order != idx).sum() > 500       # the lowest index is not the first point the search meets
        lv = settle_levels(q, t, 1, nearest=True)
        assert set(lv.tolist()) >= ({0} if spacing == 0.25 else {0, 1})


def test_selfcheck_small_targets_settle_only_on_the_final_level():
    for k in (2, 5, 16):
        for n in range(2, k):
            q, t = small_target_scene(n)
            lv = levels(*box(t))
            assert len(lv) == 4 and not lv[0]["final"]
            assert (settle_levels(q[::10], t, k) == 3).all()


def test_selfcheck_outside_scene():
    q, t = outside_scene()
    lo, hi = box(t)
    assert ((q < lo) | (q > hi)).any(1)[:-3].all()
    dk = brute_smallest(q[-14:-3], t, 2)
    assert np.isfinite(dk[:6]).all() and np.isinf(dk[6:]).all()
    with np.errstate(over="ignore"):
        assert np.isinf(avg_of(dk, 2, len(t))[6:]).all()


@pytest.mark.parametrize("length", [40000.0, 30000.0])
def test_selfcheck_corridor_levels(length):
    q, t = corridor_scene(length)
    mn, mx = box(t)
    c0 = pyramid_cell0(mn, mx)
    assert (c0 > 0.25) == (length == 40000.0)
    lv = levels(mn, mx)
    assert len(lv) == MAX_LEVELS and lv[-1]["natural"] and (lv[0]["dim"] < 2 ** CELL_BITS).all()
    near_pairs = q[-60 * ((len(t) - 60002) // 2):]
    assert (settle_levels(near_pairs[::6], t, 4) == MAX_LEVELS - 1).any()
    gaps = q[20000:24000]
    assert (settle_levels(gaps[::20], t, 1, nearest=True) == MAX_LEVELS - 1).any()


def test_selfcheck_self_mode_key_width_and_launch_cut():
    """8192 keyframes need all 13 segment bits above the 51 cell bits; 8200 keyframes go in launches of 8192 and 8
    (plan_keyframe_chunks with at most kGridMaxSegments keyframes per launch)."""
    seg_bits = 0
    while (1 << seg_bits) < MAX_SEGMENTS:
        seg_bits += 1
    assert SEG_SHIFT + seg_bits == 64 and ((MAX_SEGMENTS - 1) << SEG_SHIFT) >> 63 == 1
    _, sizes = many_keyframes(8200)
    off = offsets_of(sizes)
    cut, kf = [0], 0
    while kf < 8200:
        e = kf + 1
        while e < 8200 and e - kf < MAX_SEGMENTS and off[e + 1] - off[kf] <= 1 << 24:
            e += 1
        cut.append(e)
        kf = e
    assert cut == [0, 8192, 8200]
    kfs = ragged_keyframes()
    assert any(len(x) == 0 for x in kfs) and any(0 < len(x) < 16 for x in kfs)


def test_selfcheck_icp_side_keyframe_reaches_level_four():
    q, t = corridor_scene(40000.0)
    side = t[:3000] + [0, 120.0, 0]
    d, _ = brute_nearest(f32(side[::30]), t[:6000])
    assert (np.sqrt(d) > 100).all() and (np.sqrt(d) < 150).all()
    lv = settle_levels(f32(side[::30]), t, 1, nearest=True, chunk=8)
    assert (lv >= 4).all()
