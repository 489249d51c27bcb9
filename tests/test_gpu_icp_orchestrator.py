"""The ICP refinement through the host orchestrator (ltrh_set_icp_refinement, ltrh_icp_stats): off, every result equals a run that never
calls the setter; on, Step 2's scan sets equal ltr_icp_refine + ltr_knn_diff_refined on the orchestrator's own inputs, and a known
query-pose error leaves fewer ND / PD candidate points than without refinement."""
import numpy as np
import pytest

import oracle
from lt_mapper_b200 import removert

pytestmark = pytest.mark.gpu

SCANSETS = ["keyframe_scans_static_projected_", "scans_knn_coexist_", "scans_knn_diff_", "keyframe_scans_updated_", "keyframe_scans_pd_",
            "keyframe_scans_strong_nd_", "keyframe_scans_weak_nd_"]
CLOUDS = ["map_global_curr_static_", "map_global_nd_", "map_global_nd_strong_", "map_global_nd_weak_", "map_global_pd_",
          "map_global_pd_strong_", "map_global_pd_weak_", "map_global_updated_"]


def _rot(axis, deg):
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    R = np.eye(4)
    R[i, i] = c; R[j, j] = c; R[i, j] = -s; R[j, i] = s
    return R


def _pipeline(c, q, q_poses, icp, steps=("12", "3")):
    G = removert.Removerter(num_knn=2, knn_thr=0.01)
    if icp is not None:
        G.set_icp_refinement(icp)
    G.load_session(0, c.xyzi, c.offsets, c.poses, oracle.inverse_poses(c.poses))
    G.load_session(1, q.xyzi, q.offsets, q_poses, oracle.inverse_poses(q_poses))
    G.run_step0()
    out = {}
    for st in steps:
        getattr(G, "run_step" + st)()
        for sess in (0, 1):
            for n in SCANSETS:
                try:
                    out[(st, sess, n)] = G.scanset(n, sess)
                except Exception:  # noqa: BLE001 -- not every member exists after every step
                    pass
            for n in CLOUDS:
                try:
                    out[(st, sess, n)] = G.cloud(n, sess)
                except Exception:  # noqa: BLE001
                    pass
    return G, out


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_refinement_off_changes_nothing(small_pair):
    c, q = (s.subset(0, 4) for s in small_pair)
    G0, ref = _pipeline(c, q, q.poses, None)
    G1, off = _pipeline(c, q, q.poses, False)
    assert ref.keys() == off.keys() and len(ref) > 20
    for key in ref:
        a, b = ref[key], off[key]
        if isinstance(a, tuple):
            assert all(_same(x, y) for x, y in zip(a, b)), key
        else:
            assert _same(a, b), key
    assert G1.icp_stats(0)["fitness"].size == 0
    G0.close()
    G1.close()


def _check_composition(G, out, c, q, qp):
    """Step 2's scan sets of a refined run equal ltr_icp_refine + ltr_knn_diff_refined (accept iff fitness < 1.0) on the orchestrator's own
    inputs; returns the two sessions' icp_stats."""
    import lt_mapper_b200 as ltr
    stats = []
    with ltr.Context(device=0) as ctx:
        for sess, other, d, poses in ((0, 1, c, c.poses), (1, 0, q, qp)):
            st = G.icp_stats(sess)
            assert st["fitness"].size == d.K and (st["accepted"] == (st["fitness"] < 1.0)).all()
            scans, off = G.scanset("keyframe_scans_static_projected_", sess)
            ss = ctx.scanset_upload(scans, off)
            ps = ctx.poses_upload(poses, oracle.inverse_poses(poses))
            th = ctx.cloud_upload(G.cloud("map_global_curr_static_", other))
            td = ctx.voxel_centroid(th, 0.4)
            T, fit, it, ex = ctx.icp_refine(ss, ps, td)
            assert np.array_equal(T.view(np.uint32), st["T"].view(np.uint32)) and np.array_equal(fit, st["fitness"])
            assert np.array_equal(it, st["iterations"]) and np.array_equal(ex, st["exit"])
            co, di = ctx.knn_diff_refined(ss, ps, th, 2, 0.01, T, fit < 1.0)
            for h, name in ((co, "scans_knn_coexist_"), (di, "scans_knn_diff_")):
                a, b = ctx.scanset_download(h), out[("12", sess, name)]
                assert _same(a[0], b[0]) and np.array_equal(a[1], b[1]), (sess, name)
            stats.append(st)
    return stats


def _error(trans, deg):
    E = _rot(2, deg) @ _rot(0, deg / 3)
    E[:3, 3] = np.array([1.0, -0.6, 0.2]) * trans
    return E


def test_refinement_on_equals_the_two_calls_and_lowers_nd_pd(small_pair):
    c, q = (s.subset(0, 4) for s in small_pair)
    E = _rot(2, 1.0) @ _rot(0, 0.3)
    E[:3, 3] = [0.3, -0.2, 0.05]
    qp = np.stack([p @ E for p in q.poses])        # query poses carrying a known error
    counts = {}
    for on in (False, True):
        G, out = _pipeline(c, q, qp, on, steps=("12",))
        counts[on] = [len(out[("12", s, "scans_knn_diff_")][0]) for s in (0, 1)]
        if on:
            st = _check_composition(G, out, c, q, qp)
            assert st[1]["accepted"].any()
        G.close()
    print(f"ND / PD candidate points after Step 2 with a query-pose error: without ICP {counts[False]}, with ICP {counts[True]}")
    assert counts[True][0] < counts[False][0] and counts[True][1] < counts[False][1]


def test_rejected_keyframes_keep_the_unrefined_diff(small_pair):
    """Query poses with errors large enough that some keyframes end with fitness >= 1.0: those keep ltr_knn_diff's result while the
    accepted ones are refined, and the orchestrator still equals the two C-ABI calls.  The stats are released with Step 2's results."""
    c, q = (s.subset(0, 6) for s in small_pair)
    for trans, deg in ((2.0, 8.0), (4.0, 15.0), (8.0, 30.0), (15.0, 60.0)):
        qp = np.stack([p @ _error(trans, deg) for p in q.poses])
        G, out = _pipeline(c, q, qp, True, steps=("12",))
        st = _check_composition(G, out, c, q, qp)
        rejected = sum(int((~s["accepted"]).sum()) for s in st)
        if rejected:
            break
        G.close()
    assert rejected, "no pose error made a keyframe fail the fitness test"
    print(f"pose error {trans} m / {deg} deg: {rejected} keyframes rejected, {sum(int(s['accepted'].sum()) for s in st)} accepted")
    G.reset_to_step0()
    assert G.icp_stats(0)["fitness"].size == 0 and G.icp_stats(1)["fitness"].size == 0
    G.close()
