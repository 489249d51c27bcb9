"""LT-map change composition and map rollback on the device: ltr_knn_split_per_keyframe bit for bit against the CPU restatement
(tests/_delta_oracle.py), and the orchestrator's delta maps (ltrh_set_delta_maps, ltrh_compose_changes, ltrh_rollback) over a
three-session in-memory cascade."""
import numpy as np
import pytest

import oracle
import _delta_oracle as D
import lt_mapper_b200 as ltr
from lt_mapper_b200 import removert

pytestmark = pytest.mark.gpu


def _same(a, b):
    a = np.asarray(a, np.float32).reshape(-1, 4); b = np.asarray(b, np.float32).reshape(-1, 4)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _split_device(ctx, Q, T, k, thr):
    """(near, far) per keyframe from the device."""
    q = ctx.scanset_upload(*D.pack(Q))
    t = ctx.scanset_upload(*D.pack(T))
    try:
        n, f = ctx.knn_split_per_keyframe(q, t, k, thr)
    finally:
        ctx.scanset_free(q); ctx.scanset_free(t)
    out = []
    for h in (n, f):
        pts, off = ctx.scanset_download(h)
        out.append(D.split_sets(pts, off))
        ctx.scanset_free(h)
    return out


def _check(ctx, Q, T, k, thr):
    near, far = _split_device(ctx, Q, T, k, thr)
    assert len(near) == len(Q) == len(far)
    for j, (q, t) in enumerate(zip(Q, T)):
        m = D.far_mask(q, t, k, thr)
        assert _same(far[j], np.asarray(q, np.float32).reshape(-1, 4)[m]), (j, k)
        assert _same(near[j], np.asarray(q, np.float32).reshape(-1, 4)[~m]), (j, k)
    return sum(len(f) for f in far), sum(len(n) for n in near)


def _random_sets(rng, K, sizes_t, scale=2.0, n_q=200, dup=True):
    Q, T = [], []
    for j in range(K):
        c = rng.normal(0, 50, 3)
        q = np.concatenate([c + rng.random((n_q, 3)) * scale, rng.random((n_q, 1))], 1).astype(np.float32)
        if dup:
            q[: n_q // 10] = q[n_q // 10: 2 * (n_q // 10)]          # duplicated points
        nt = sizes_t[j % len(sizes_t)]
        src = q[rng.integers(0, n_q, nt)]
        t = src + np.concatenate([rng.normal(0, 0.04, (nt, 3)), np.zeros((nt, 1))], 1).astype(np.float32)
        Q.append(q); T.append(t)
    return Q, T


@pytest.fixture(scope="module")
def ctx():
    c = ltr.Context()
    yield c
    c.close()


def test_split_random_sets_every_k(ctx):
    """k = 1..16 with target keyframes of 0, 1, k - 1, k and many points, duplicates in the queries, an empty query keyframe."""
    rng = np.random.default_rng(7)
    for k in range(1, 17):
        Q, T = _random_sets(rng, 7, [0, 1, max(k - 1, 0), k, 150, 400, 150])
        Q[6] = Q[6][:0]                                              # an empty query keyframe
        T[5] = np.repeat(Q[5][:50], 16, 0)                           # every one of the first 50 queries has >= k targets at distance 0
        thr = float(np.float32([0.01, 0.004, 0.02][k % 3]))
        nf, nn = _check(ctx, Q, T, k, thr)
        assert nf > 0 and nn >= 50, k


def test_split_pipeline_shaped(ctx, cascade):
    """Scans of a finished pair against their own PD and strong-ND sets, the shapes composition and rollback feed the primitive."""
    g0 = cascade["gen"][0]
    for q, t in (("static", "pd"), ("static", "nd"), ("nd", "pd"), ("pd", "nd"), ("live0", "pd")):
        for k, thr in ((2, 0.01), (1, 0.04)):
            _check(ctx, g0[q], g0[t], k, thr)


def test_split_extent_forces_cell_growth(ctx):
    """Targets 2e5 m apart in one keyframe: the 0.14 m reach would need far more than 2^17 cells per axis, so the cell grows."""
    rng = np.random.default_rng(11)
    Q, T = _random_sets(rng, 3, [300], n_q=300)
    for j in range(3):
        far = Q[j].copy(); far[:, 0] += 2e5
        Q[j] = np.concatenate([Q[j], far]); T[j] = np.concatenate([T[j], T[j] + np.array([2e5, 0, 0, 0], np.float32)])
    nf, nn = _check(ctx, Q, T, 2, 0.01)
    assert nf > 0 and nn > 0


def test_split_many_keyframes_and_tiny_launches(ctx, monkeypatch):
    """More than 8192 keyframes (the level's segment limit), then a points-per-launch knob small enough to force one launch per keyframe."""
    rng = np.random.default_rng(5)
    Q, T = _random_sets(rng, 9000, [0, 1, 3, 12], n_q=6, scale=0.3, dup=False)
    launches0 = ctx.kernel_launches()
    _check(ctx, Q, T, 3, 0.01)
    wide = ctx.kernel_launches() - launches0
    monkeypatch.setenv("LTR_DELTA_CHUNK_POINTS", "7")
    Q2, T2 = Q[:300], T[:300]
    launches0 = ctx.kernel_launches()
    _check(ctx, Q2, T2, 3, 0.01)
    assert ctx.kernel_launches() - launches0 >= 300 > wide


def test_split_rejects_non_finite_without_leaks(ctx):
    rng = np.random.default_rng(2)
    Q, T = _random_sets(rng, 3, [40])
    live0 = ctx.memory_stats()[0]
    for bad_q in (True, False):
        for v in (np.nan, np.inf):
            Qb = [q.copy() for q in Q]; Tb = [t.copy() for t in T]
            (Qb if bad_q else Tb)[1][3, 1] = v
            q = ctx.scanset_upload(*D.pack(Qb)); t = ctx.scanset_upload(*D.pack(Tb))
            with pytest.raises(ltr.LtrError) as e:
                ctx.knn_split_per_keyframe(q, t, 2, 0.01)
            assert e.value.code == -3
            ctx.scanset_free(q); ctx.scanset_free(t)
            assert ctx.memory_stats()[0] == live0
    q = ctx.scanset_upload(*D.pack(Q)); t = ctx.scanset_upload(*D.pack(T[:2]))
    with pytest.raises(ltr.LtrError):                  # keyframe counts differ
        ctx.knn_split_per_keyframe(q, t, 2, 0.01)
    ctx.scanset_free(q); ctx.scanset_free(t)
    assert ctx.memory_stats()[0] == live0


def test_split_live_bytes_back_to_baseline(ctx):
    rng = np.random.default_rng(9)
    Q, T = _random_sets(rng, 40, [0, 5, 300])
    q = ctx.scanset_upload(*D.pack(Q)); t = ctx.scanset_upload(*D.pack(T))
    live0 = ctx.memory_stats()[0]
    n, f = ctx.knn_split_per_keyframe(q, t, 4, 0.01)
    ctx.scanset_free(n); ctx.scanset_free(f)
    assert ctx.memory_stats()[0] == live0
    ctx.scanset_free(q); ctx.scanset_free(t)


# ---- orchestrator --------------------------------------------------------------------------------------------------------------------
def _grid(d):   # Session::loadKeyframes' pcl::VoxelGrid (Session.cpp:284-289) on every scan
    sc = [removert.voxel_grid(d.scan(k), 0.05)[0] for k in range(d.K)]
    return D.pack(sc)


def _sets(G, name):
    return D.split_sets(*G.scanset(name, 0))


@pytest.fixture(scope="module")
def cascade():
    """Sessions 0 -> 1 -> 2 of synth promoted in memory with delta maps on.  Session 2 has every car, so it brings back the cars session
    1 removed: generation 1's PD cancels part of generation 0's ND."""
    import synth
    K = 4
    sess = [synth.make_session(s, K, beams=32, az_steps=900) for s in (0, 1, 2)]
    loaded = [_grid(d) for d in sess]
    inv = [oracle.inverse_poses(d.poses) for d in sess]
    G = removert.Removerter(num_knn=2, knn_thr=0.01)
    G.set_delta_maps(True)
    G.load_session(0, *loaded[0], sess[0].poses, inv[0])
    gen = []
    for g in (1, 2):
        G.load_session(1, *loaded[g], sess[g].poses, inv[g])
        live = _sets(G, "keyframe_scans_")
        G.run_step0(); G.run_step12(); G.run_step3()
        gen.append({"pd": _sets(G, "keyframe_scans_pd_"), "nd": _sets(G, "keyframe_scans_strong_nd_"),
                    "static": _sets(G, "keyframe_scans_static_projected_"), "live0": live})
        G.cascade_promote_updated()
    out = {"G": G, "gen": gen, "poses": sess[0].poses, "inv": inv[0], "live": _sets(G, "keyframe_scans_"), "loaded0": loaded[0]}
    yield out
    G.close()


def test_recorded_deltas_are_the_generations_sets(cascade):
    G = cascade["G"]
    assert G.delta_count() == 2
    for g in (0, 1):
        G.compose_changes(g, g + 1)
        assert all(_same(a, b) for a, b in zip(_sets(G, "composed_pd_"), cascade["gen"][g]["pd"]))
        assert all(_same(a, b) for a, b in zip(_sets(G, "composed_nd_"), cascade["gen"][g]["nd"]))


def test_compose_and_rollback_match_the_oracle(cascade):
    G, gen = cascade["G"], cascade["gen"]
    deltas = [(x["pd"], x["nd"]) for x in gen]
    G.compose_changes(0, 2)
    pd, nd = D.compose(deltas, 0, 2, 2, 0.01)
    assert all(_same(a, b) for a, b in zip(_sets(G, "composed_pd_"), pd))
    assert all(_same(a, b) for a, b in zip(_sets(G, "composed_nd_"), nd))
    assert sum(map(len, nd)) < sum(map(len, gen[0]["nd"])) + sum(map(len, gen[1]["nd"]))     # cancellation happened
    for i in (0, 1, 2):
        G.rollback(i)
        want = D.rollback(cascade["live"], deltas, i, 2, 0.01)
        got = _sets(G, "keyframe_scans_restored_")
        assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want)), i
        assert _same(G.cloud("saved:restored_map"), D.merged_map(want, cascade["poses"])), i


def _share_far(A, B, r=0.2):
    """symmetric share of the points of A and B farther than r from the other cloud, over all keyframes"""
    from scipy.spatial import cKDTree
    n_far = n_all = 0
    for a, b in zip(A, B):
        for x, y in ((a, b), (b, a)):
            if len(x) == 0:
                continue
            n_all += len(x)
            n_far += len(x) if len(y) == 0 else int((cKDTree(y[:, :3]).query(x[:, :3])[0] > r).sum())
    return n_far / max(n_all, 1)


def test_rollback_is_closer_to_the_earlier_session(cascade):
    G = cascade["G"]
    G.rollback(0)
    restored = _sets(G, "keyframe_scans_restored_")
    ref = cascade["gen"][0]["static"]
    q_restored, q_live = _share_far(restored, ref), _share_far(cascade["live"], ref)
    print(f"share of points > 0.2 m from generation 0's static scans: restored {q_restored:.4f}, live {q_live:.4f}")
    assert q_restored < q_live


def test_delta_map_errors():
    G = removert.Removerter()
    try:
        with pytest.raises(ltr.LtrError):
            G.compose_changes(0, 1)          # delta maps off
        with pytest.raises(ltr.LtrError):
            G.rollback(0)
        with pytest.raises(ltr.LtrError):
            G.delta_load(np.zeros((0, 4)), [0], np.zeros((0, 4)), [0])
        G.load_session(0, np.array([[1, 2, 3, 0]], np.float32), np.array([0, 1], np.int64), np.eye(4)[None], np.eye(4)[None])
        G.set_delta_maps(True)
        G.delta_load(np.zeros((0, 4)), [0, 0], np.zeros((0, 4)), [0, 0])
        assert G.delta_count() == 1
        for i, j in ((0, 0), (1, 1), (0, 2), (-1, 1)):
            with pytest.raises(ltr.LtrError):
                G.compose_changes(i, j)
        for i in (-1, 2):
            with pytest.raises(ltr.LtrError):
                G.rollback(i)
        G.compose_changes(0, 1)
        G.rollback(1)
        G.rollback(0)
        G.set_delta_maps(False)
        assert G.delta_count() == 0
        with pytest.raises(ltr.LtrError):
            G.rollback(0)
    finally:
        G.close()


# ---- driver --------------------------------------------------------------------------------------------------------------------------
def test_driver_compose_matches_in_memory(tmp_path):
    """Two cascade generations through files (the driver's own scans_updated/ becomes the next central session), then --compose over both
    output trees == the same delta maps loaded and composed through the orchestrator in memory."""
    import os
    import shutil
    import subprocess
    import synth
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    binary = os.path.join(root, "lt_mapper_b200", "ltremovert_b200")
    K = 4
    for name, s in zip("abc", [synth.make_session(s, K, beams=32, az_steps=900) for s in (0, 1, 2)]):
        os.makedirs(tmp_path / name / "Scans")
        with open(tmp_path / name / "poses.txt", "w") as f:
            for k in range(s.K):
                removert.write_pcd(str(tmp_path / name / "Scans" / f"{k:06d}.pcd"), s.scan(k))
                f.write(" ".join(repr(float(v)) for v in s.poses[k][:3].ravel()) + "\n")
    ident = [1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0]

    def run(central_scans, query, out, *extra):
        cfg = tmp_path / f"params_{query}_{len(extra)}.yaml"
        cfg.write_text("removert:\n  saveMapPCD: true\n" + f'  save_pcd_directory: "{out}"\n'
                       + f'  central_sess_scan_dir: "{central_scans}"\n  central_sess_pose_path: "{tmp_path}/a/poses.txt"\n'
                       + f'  query_sess_scan_dir: "{tmp_path}/{query}/Scans/"\n  query_sess_pose_path: "{tmp_path}/{query}/poses.txt"\n'
                       + "  ExtrinsicLiDARtoPoseBase: [" + ", ".join(repr(v) for v in ident) + "]\n"
                       + "  keyframe_gap: 1\n  start_idx: 0\n  end_idx: 100\n  downsample_voxel_size: 0.05\n"
                       + "  num_nn_points_within: 2\n  dist_nn_points_within: 0.01\n")
        return subprocess.run([binary, "--config", str(cfg), *extra], capture_output=True, text=True, timeout=600)

    r = run(tmp_path / "a" / "Scans", "b", tmp_path / "out1")
    assert r.returncode == 0, r.stdout + r.stderr
    shutil.copytree(tmp_path / "out1" / "scans_updated", tmp_path / "central2")
    r = run(tmp_path / "central2", "c", tmp_path / "out2")
    assert r.returncode == 0, r.stdout + r.stderr
    shutil.copytree(tmp_path / "out2" / "scans_updated", tmp_path / "central3")
    r = run(tmp_path / "central3", "c", tmp_path / "out3", f"--compose={tmp_path}/out1,{tmp_path}/out2")
    assert r.returncode == 0, r.stdout + r.stderr
    names = sorted(os.listdir(tmp_path / "out2" / "scans_pd"))
    assert names and sorted(os.listdir(tmp_path / "out3" / "composed" / "scans_restored")) == names

    # in memory, from the same files
    idx = [int(n.split(".")[0]) for n in names]
    poses = removert.read_poses(str(tmp_path / "a" / "poses.txt"))[idx]
    live = D.pack([removert.read_pcd(str(tmp_path / "central3" / n)) for n in names])
    G = removert.Removerter(num_knn=2, knn_thr=0.01)
    try:
        G.load_session_raw(0, *live, poses, oracle.inverse_poses(poses))
        G.set_delta_maps(True)
        for out in ("out1", "out2"):
            G.delta_load(*D.pack([removert.read_pcd(str(tmp_path / out / "scans_pd" / n)) for n in names]),
                         *D.pack([removert.read_pcd(str(tmp_path / out / "scans_nd_strong" / n)) for n in names]))
        G.compose_changes(0, 2)
        G.rollback(0)
        for sub, sname in (("scans_pd", "composed_pd_"), ("scans_nd_strong", "composed_nd_"), ("scans_restored", "keyframe_scans_restored_")):
            got = _sets(G, sname)
            for k, n in enumerate(names):
                assert _same(removert.read_pcd(str(tmp_path / "out3" / "composed" / sub / n)), got[k]), (sub, n)
        assert _same(removert.read_pcd(str(tmp_path / "out3" / "composed" / "restored_map.pcd")), G.cloud("saved:restored_map"))
    finally:
        G.close()
    for flag in ("--selfremovert", "--clean-scans", "--icp-refinement", "--adaptive-threshold", "--map-ball"):   # they configure Steps 0-3
        r = run(tmp_path / "central3", "c", tmp_path / "out5", f"--compose={tmp_path}/out1", flag)
        assert r.returncode == 2 and "--compose" in r.stderr, (flag, r.stderr)
    os.remove(tmp_path / "out1" / "scans_pd" / names[1])
    r = run(tmp_path / "central3", "c", tmp_path / "out4", f"--compose={tmp_path}/out1,{tmp_path}/out2")
    assert r.returncode != 0 and os.path.join("scans_pd", names[1]) in r.stderr
