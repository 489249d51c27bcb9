"""The ball-subset restatement (tests/_ball_oracle.py) on the CPU: its membership rule against a float64 distance away from the sphere,
at the sphere to the ulp, for non-finite points, and the composition against the oracle's full pass when every point is in every ball."""
import numpy as np
import pytest

import oracle
import _ball_oracle as B

F32 = np.float32


def test_membership_agrees_with_float64_away_from_the_boundary():
    rng = np.random.default_rng(7)
    c = np.array([12.25, -40.5, 1.75], F32)
    p = (c + rng.normal(0.0, 60.0, (200_000, 3))).astype(F32)
    for radius in (0.5, 13.0, 80.0, 250.0):
        d2 = ((p.astype(np.float64) - c.astype(np.float64)) ** 2).sum(1)
        r2 = np.float64(radius) ** 2
        away = np.abs(d2 - r2) > 1e-5 * r2
        got = B.members(p, c, radius)
        assert away.sum() > 0.99 * len(p)
        assert np.array_equal(got[away], (d2 < r2)[away]), radius


def test_membership_at_the_sphere_to_the_ulp():
    """d2 equal to r2 is outside, one ulp below is inside (the strict test of FLANN's RadiusResultSet)."""
    rng = np.random.default_rng(3)
    c = np.array([5.5, -3.25, 0.5], F32)
    checked = 0
    for _ in range(200):
        p = (c + rng.normal(0.0, 20.0, (1, 3))).astype(F32)
        d2 = B.sq_dist(p, c)[0]
        for r2, inside in ((d2, False), (np.nextafter(d2, F32(np.inf)), True)):
            R = F32(np.sqrt(np.float64(r2)))
            if B.radius2(R) != r2:
                continue
            assert bool(B.members(p, c, R)[0]) == inside, (p, c, R)
            checked += 1
    assert checked > 100


def test_non_finite_points_are_never_members():
    c = np.zeros(3, F32)
    p = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1, 1, 1]], F32)
    assert B.members(p, c, 1e30).tolist() == [False, False, False, True]


@pytest.mark.parametrize("mode", [oracle.MODE_HD, oracle.MODE_ND, oracle.MODE_PD])
def test_a_ball_around_everything_is_the_full_pass(small_pair, small_maps, mode):
    c = small_pair[0]
    m = small_maps[0] if mode == oracle.MODE_HD else small_maps[1][::7]
    inv = oracle.inverse_poses(c.poses)
    full = oracle.remove_pass(m, c.xyzi, c.offsets, inv, mode, 2.5)
    ball = B.remove_pass(m, c.xyzi, c.offsets, c.poses, inv, mode, 2.5, 1e6)
    assert full.sum() > 0 and np.array_equal(ball, full)
    # a ball that cuts the map changes the flags
    d = np.sqrt(B.sq_dist(m, B.centres(c.poses)[0]).astype(np.float64))
    R = float(np.quantile(d, 0.5))
    one = B.remove_pass(m, c.xyzi, c.offsets[:2], c.poses[:1], inv[:1], mode, 2.5, R)
    assert not np.array_equal(one, oracle.remove_pass(m, c.xyzi, c.offsets[:2], inv[:1], mode, 2.5))
