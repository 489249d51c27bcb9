"""The range-adaptive discrepancy threshold on the CPU: the per-pixel rule of tests/_adaptive_oracle.py pinned against a scalar float32
restatement of calcDescrepancyAndParseDynamicPointIdx (Removerter.cpp:388-410) with line 396 in place of line 398, the restated pass
pinned against the oracle's own pass with the threshold folded back to a constant, and known answers at the edges of the rule."""
import numpy as np
import pytest

import oracle
import _adaptive_oracle as A

F32 = np.float32


def _reference_loop(scan_rimg, map_rimg, ptidx, mode, coeff):
    """Removerter.cpp:388-410, one pixel at a time in row-major order, with
        float adaptive_coeff = coeff;                                                    // :395
        float adaptive_dynamic_descrepancy_threshold = adaptive_coeff * this_range;     // :396
    and the diff image of the variant (scan - map :572 / :459, map - scan :516)."""
    out = []
    for r in range(scan_rimg.shape[0]):
        for c in range(scan_rimg.shape[1]):
            s, m = F32(scan_rimg[r, c]), F32(map_rimg[r, c])
            this_diff = F32(m - s) if mode == oracle.MODE_ND else F32(s - m)
            this_range = s
            thres = F32(F32(coeff) * this_range)
            if this_diff < F32(200.0) and this_diff > thres:
                out.append(int(ptidx[r, c]))
    return out


def _random_images(rng, rows, cols):
    s = rng.uniform(0.5, 120.0, (rows, cols)).astype(F32)
    m = (s * rng.uniform(0.3, 1.7, (rows, cols))).astype(F32)
    s[rng.random((rows, cols)) < 0.15] = F32(10000.0)                 # no scan return
    m[rng.random((rows, cols)) < 0.15] = F32(10000.0)                 # no map point
    edge = rng.random((rows, cols)) < 0.2                             # diff exactly at, one ulp below and above the threshold
    t = (F32(0.05) * s).astype(F32)
    m_edge = (s - t).astype(F32)
    m_edge = np.where(rng.random((rows, cols)) < 0.5, np.nextafter(m_edge, F32(np.inf)), m_edge)
    m[edge] = m_edge[edge]
    return s, m


@pytest.mark.parametrize("mode", [oracle.MODE_HD, oracle.MODE_ND, oracle.MODE_PD])
@pytest.mark.parametrize("coeff", [0.01, 0.05, 0.2, 0.95])
def test_pixel_rule_matches_the_reference_loop(mode, coeff):
    rng = np.random.default_rng(17 + mode)
    rows, cols = 24, 61
    s, m = _random_images(rng, rows, cols)
    ptidx = rng.integers(0, 1 << 20, (rows, cols)).astype(np.int32)
    exp = _reference_loop(s, m, ptidx, mode, coeff)
    got = ptidx[A.pixel_flags(s, m, mode, coeff)].tolist()
    assert got == exp
    if coeff < 0.9:
        assert len(exp) > 0


def test_restated_pass_equals_the_oracle_pass_with_a_constant(small_pair, small_maps, monkeypatch):
    """The pass around the rule is the oracle's: with the per-pixel threshold replaced by the constant 0.1, the restatement gives the
    oracle's flags bit for bit (HD, PD, ND)."""
    c = small_pair[0]
    inv = oracle.inverse_poses(c.poses)

    def constant_rule(scan_rimg, map_rimg, mode, coeff):
        s, m = np.asarray(scan_rimg, F32), np.asarray(map_rimg, F32)
        diff = (m - s) if mode == oracle.MODE_ND else (s - m)
        return (diff < F32(200.0)) & (diff > F32(0.1))

    monkeypatch.setattr(A, "pixel_flags", constant_rule)
    for mode, m in ((oracle.MODE_HD, small_maps[0]), (oracle.MODE_PD, small_maps[1][::7]), (oracle.MODE_ND, small_maps[1][::7])):
        exp = oracle.remove_pass(m, c.xyzi, c.offsets, inv, mode, 2.5)
        got = A.remove_pass(m, c.xyzi, c.offsets, inv, mode, 2.5, None)
        assert np.array_equal(got, exp), mode
        assert exp.sum() > 0


# ------------------------------------------------------------------------------------------------------------ known answers
def _on_axis(r):
    """A point at range r straight ahead (azimuth 0, elevation 0): its range is sqrt(fl(r * r)) == r."""
    return np.array([[r, 0.0, 0.0, 1.0]], F32)


def _one(scan_r, map_r, mode, coeff):
    I = np.eye(4)[None]
    scan = _on_axis(scan_r) if scan_r is not None else np.zeros((0, 4), F32)
    return int(A.remove_pass(_on_axis(map_r), scan, np.array([0, len(scan)], np.int64), I, mode, 2.5, coeff)[0])


def threshold_edge(s, coeff):
    """The floats rho around the edge of the rule at scan range s: the map ranges whose fl(s - rho) are the last above and the first at
    or below t = fl(coeff s), in increasing range order."""
    s, t = F32(s), F32(F32(coeff) * F32(s))
    rho = np.nextafter(F32(s - t), F32(-np.inf))
    for _ in range(8):
        rho = np.nextafter(rho, F32(-np.inf))
    while not F32(s - np.nextafter(rho, F32(np.inf))) <= t:
        rho = np.nextafter(rho, F32(np.inf))
    return rho, np.nextafter(rho, F32(np.inf))


def test_known_answer_at_the_threshold():
    """s = 4, c = 0.05: t = fl(0.2).  Of the two consecutive map ranges on either side of the edge, the nearer one (fl(4 - rho) > t)
    flags and the farther one does not.  The constant 0.1 flags both."""
    s, coeff = 4.0, 0.05
    t = F32(F32(coeff) * F32(s))
    assert t == F32(0.2)
    inside, outside = threshold_edge(s, coeff)
    assert F32(F32(s) - inside) > t >= F32(F32(s) - outside)
    for mode in (oracle.MODE_HD, oracle.MODE_PD):
        assert [_one(s, r, mode, coeff) for r in (inside, outside)] == [1, 0]
    assert all(F32(F32(s) - r) > F32(0.1) for r in (inside, outside))


def test_known_answer_diff_equal_to_the_threshold():
    """The inequality is strict: s = 4, c = 2^-4 gives t = 0.25 exactly, and rho = 3.75 has fl(4 - rho) == t: no flag; one ulp nearer
    (diff one ulp of 4 above t) flags, one ulp farther does not."""
    s, coeff = 4.0, 0.0625
    t = F32(F32(coeff) * F32(s))
    rho = F32(3.75)
    assert F32(F32(s) - rho) == t
    for mode in (oracle.MODE_HD, oracle.MODE_PD):
        assert _one(s, rho, mode, coeff) == 0
        assert _one(s, np.nextafter(rho, F32(-np.inf)), mode, coeff) == 1
        assert _one(s, np.nextafter(rho, F32(np.inf)), mode, coeff) == 0


def test_known_answer_nd_sign():
    """ND compares map - scan: s = 10, c = 0.05, t = 0.5.  A map point 0.6 m behind the return flags in ND only, one 0.6 m in front in
    HD / PD only, and 0.4 m either way in neither."""
    s, c = 10.0, 0.05
    assert [_one(s, 10.6, m, c) for m in (oracle.MODE_ND, oracle.MODE_HD, oracle.MODE_PD)] == [1, 0, 0]
    assert [_one(s, 9.4, m, c) for m in (oracle.MODE_ND, oracle.MODE_HD, oracle.MODE_PD)] == [0, 1, 1]
    assert [_one(s, r, m, c) for r in (10.4, 9.6) for m in (oracle.MODE_ND, oracle.MODE_HD)] == [0, 0, 0, 0]


def test_known_answer_empty_scan_pixel():
    """No scan return: s = 10000, t = 500; scan - map > 200 for every map point within 9800 m and map - scan < 0, so nothing flags."""
    for mode in (oracle.MODE_HD, oracle.MODE_ND, oracle.MODE_PD):
        for c in (0.01, 0.05, 0.2):
            assert _one(None, 5.0, mode, c) == 0


def test_known_answer_diff_upper_bound():
    """diff >= 200 never flags whatever t is: s = 250, map at 40 (diff 210 > t = 12.5) does not flag, map at 50.5 (diff 199.5) does;
    with c = 0.9 (t = 225 > 200) nothing flags."""
    assert _one(250.0, 40.0, oracle.MODE_HD, 0.05) == 0
    assert _one(250.0, 50.5, oracle.MODE_HD, 0.05) == 1
    assert _one(250.0, 50.5, oracle.MODE_HD, 0.9) == 0
    assert _one(250.0, 40.0, oracle.MODE_HD, 0.9) == 0
