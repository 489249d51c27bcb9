"""The CPU restatement of LT-map change composition and map rollback (tests/_delta_oracle.py) on hand-built clouds: the algebra the
device path is held to (DESIGN.md §5.3)."""
import numpy as np

import _delta_oracle as D

K, THR = 1, 0.01   # one neighbour: the lattices below are sparse, so a point matches only its own copy


def _same(a, b):
    a = np.asarray(a, np.float32).reshape(-1, 4); b = np.asarray(b, np.float32).reshape(-1, 4)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _same_sets(A, B):
    return len(A) == len(B) and all(_same(a, b) for a, b in zip(A, B))


def _lattice(x0, n, step=0.5, seed=0):
    """n points, each alone in its 0.05 m voxel (so V keeps them exactly), starting at x = x0."""
    rng = np.random.default_rng(seed)
    i = np.arange(n)
    p = np.stack([x0 + step * (i % 4), step * ((i // 4) % 4), step * (i // 16), rng.random(n)], 1).astype(np.float32)
    return p + np.float32(0.0125) * np.array([1, 1, 1, 0], np.float32)     # away from the voxel walls


def _empty():
    return np.zeros((0, 4), np.float32)


def test_minus_kdtree_matches_brute_force():
    rng = np.random.default_rng(3)
    for k in (1, 2, 5, 16):
        for nb in (1, k - 1, k, 40):
            if nb < 1:
                continue
            a = (rng.random((300, 4)) * [2, 2, 2, 1]).astype(np.float32)
            b = np.concatenate([a[rng.choice(300, min(nb, 300), replace=False)] + rng.normal(0, 0.05, (min(nb, 300), 4)).astype(np.float32),
                                (rng.random((max(nb - 300, 0), 4))).astype(np.float32)])[:nb]
            assert np.array_equal(D.far_mask(a, b, k, THR), D.far_mask(a, b, k, THR, brute=True)), (k, nb)


def test_empty_target_keeps_everything_and_order():
    a = _lattice(0.0, 20)
    assert _same(D.minus(a, _empty(), K, THR), a)
    assert _same(D.minus(a[::-1], a[:3], K, THR), a[::-1][:-3])


def test_small_target_divides_by_k():
    # one target point at distance^2 0.015: k = 1 -> 0.015 >= 0.01 far; k = 2 -> 0.0075 < 0.01 near (the sum is still divided by k)
    a = np.array([[0.0, 0.0, 0.0, 0.0]], np.float32)
    b = np.array([[np.sqrt(np.float32(0.015)), 0.0, 0.0, 0.0]], np.float32)
    assert D.far_mask(a, b, 1, THR)[0] and not D.far_mask(a, b, 2, THR)[0]


def test_mean_exactly_on_threshold_is_far():
    q = np.array([[0.1, 0.0, 0.0, 0.0]], np.float32)
    t = np.zeros((1, 4), np.float32)
    d = np.float32(q[0, 0]) * np.float32(q[0, 0])      # L2_Simple of (0.1, 0, 0) in f32
    assert D.far_mask(q, t, 1, d)[0]
    assert not D.far_mask(q, t, 1, np.nextafter(d, np.float32(1)))[0]


def test_one_generation_returns_the_recorded_delta():
    pd, nd = [_lattice(20.0, 8), _empty()], [_lattice(10.0, 5), _lattice(30.0, 3)]
    cpd, cnd = D.compose([(pd, nd)], 0, 1, K, THR)
    assert _same_sets(cpd, pd) and _same_sets(cnd, nd)


def test_empty_deltas_are_the_identity_up_to_v():
    live = [_lattice(0.0, 30, seed=1), _empty(), np.repeat(_lattice(5.0, 4), 3, 0)]   # duplicates collapse under V
    E = [_empty() for _ in live]
    out = D.rollback(live, [(E, E), (E, E)], 0, K, THR)
    assert _same_sets(out, D.V(live))
    assert _same_sets(D.rollback(live, [(E, E)], 1, K, THR), live)


def test_remove_then_readd_cancels():
    car = _lattice(10.0, 12)
    E = [_empty()]
    pd, nd = D.compose([(E, [car]), ([car], E)], 0, 2, K, THR)
    assert len(pd[0]) == 0 and len(nd[0]) == 0


def test_add_then_remove_cancels():
    car = _lattice(20.0, 12)
    E = [_empty()]
    pd, nd = D.compose([([car], E), (E, [car])], 0, 2, K, THR)
    assert len(pd[0]) == 0 and len(nd[0]) == 0


def test_separated_geometry_is_restored_exactly():
    static, car_a, car_b, car_c = _lattice(0.0, 40, seed=2), _lattice(10.0, 16, seed=3), _lattice(20.0, 16, seed=4), _lattice(30.0, 16, seed=5)
    s0 = [np.concatenate([static, car_a])]
    s1 = [np.concatenate([static, car_b])]          # generation 0: car A removed, car B added
    s2 = [np.concatenate([static, car_b, car_c])]   # generation 1: car C added
    deltas = [([car_b], [car_a]), ([car_c], [_empty()])]
    live = D.V(s2)
    assert _same_sets(D.rollback(live, deltas, 0, K, THR), D.V(s0))
    assert _same_sets(D.rollback(live, deltas, 1, K, THR), D.V(s1))
    assert _same_sets(D.rollback(live, deltas, 2, K, THR), live)
    pd, nd = D.compose(deltas, 0, 2, K, THR)
    assert _same_sets(pd, D.V([np.concatenate([car_b, car_c])])) and _same_sets(nd, D.V([car_a]))
