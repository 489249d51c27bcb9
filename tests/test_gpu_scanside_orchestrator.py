"""Scan-side removal through the host orchestrator (ltrh_scanside_removal) and the drop-in driver (--clean-scans), against the CPU
restatement (tests/_scanside_oracle.py) on the orchestrator's own inputs, byte for byte; a 2-rank driver run equals the single-process
one when two GPUs are visible."""
import os
import subprocess

import numpy as np
import pytest

import oracle
import _scanside_oracle as so
from lt_mapper_b200 import removert

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "lt_mapper_b200", "ltremovert_b200")


def _n_gpus():
    try:
        import torch
        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:  # noqa: BLE001
        return 0


def _per_kf(pts, off):
    return [pts[off[j]:off[j + 1]] for j in range(len(off) - 1)]


def test_orchestrator_session_pairs_match_the_oracle(small_pair):
    c, q = (s.subset(0, 4) for s in small_pair)
    G = removert.Removerter(num_knn=3, knn_thr=0.1)
    for s, d in ((0, c), (1, q)):
        G.load_session(s, d.xyzi, d.offsets, d.poses, oracle.inverse_poses(d.poses))
    G.run_step0()
    G.run_step12()
    for crit in (so.MAP, so.SCAN_MINUS_MAP):
        for m_sess, s_sess in ((0, 0), (1, 1), (0, 1), (1, 0)):
            d = (c, q)[s_sess]
            G.scanside_removal(m_sess, s_sess, crit)
            scans, off = G.scanset("keyframe_scans_", s_sess)          # after precleaningKeyframes
            m = G.cloud("map_global_curr_static_", m_sess)
            inv = oracle.inverse_poses(d.poses)
            exp = so.split_session(scans, off, d.poses, inv, m, crit, 3, 0.1)
            for part, name in enumerate(("scans_static_", "scans_dynamic_")):
                got = _per_kf(*G.scanset(name, s_sess))
                assert len(got) == d.K
                for kf, (a, b) in enumerate(zip(got, exp[part])):
                    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), (crit, m_sess, s_sess, name, kf)
    G.reset_to_step0()     # releases the results
    with pytest.raises(Exception):
        G.scanset_handle("scans_static_", 0)
    G.close()


_PARAMS = """removert:
  saveMapPCD: true
  save_pcd_directory: "{out}"
  central_sess_scan_dir: "{d}/central/Scans/"
  central_sess_pose_path: "{d}/central/poses.txt"
  query_sess_scan_dir: "{d}/query/Scans/"
  query_sess_pose_path: "{d}/query/poses.txt"
  sequence_vfov: 50
  sequence_hfov: 360
  ExtrinsicLiDARtoPoseBase: [1.0, 0.0, 0.0, 0.0,
                             0.0, 1.0, 0.0, 0.0,
                             0.0, 0.0, 1.0, 0.0,
                             0.0, 0.0, 0.0, 1.0]
  keyframe_gap: 1
  start_idx: 2
  end_idx: 5
  remove_resolution_list: [2.5]
  downsample_voxel_size: 0.05
  num_nn_points_within: 3
  dist_nn_points_within: 0.1
"""


def _dataset(tmp_path, small_pair):
    for name, sess in zip(("central", "query"), small_pair):
        d = tmp_path / name
        os.makedirs(d / "Scans", exist_ok=True)
        with open(d / "poses.txt", "w") as f:
            for k in range(sess.K):
                removert.write_pcd(str(d / "Scans" / f"{k:06d}.pcd"), sess.scan(k))
                f.write(" ".join(repr(float(v)) for v in sess.poses[k][:3].ravel()) + "\n")


def _run(tmp_path, tag, args, env=None, world=1):
    out = tmp_path / f"out_{tag}"
    cfg = tmp_path / f"params_{tag}.yaml"
    cfg.write_text(_PARAMS.format(out=out, d=tmp_path))
    if world == 1:
        r = subprocess.run([BIN, "--config", str(cfg)] + args, capture_output=True, text=True, timeout=600, env=env)
        assert r.returncode == 0, r.stdout + r.stderr
    else:
        procs = []
        for rank in range(world):
            e = dict(os.environ, RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), LTR_NCCL_ID_FILE=str(tmp_path / f"nccl_{tag}"))
            procs.append(subprocess.Popen([BIN, "--config", str(cfg)] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=e))
        for p in procs:
            o, _ = p.communicate(timeout=600)
            assert p.returncode == 0, o
    return out


def _tree(d):
    return {os.path.relpath(os.path.join(r, f), d): open(os.path.join(r, f), "rb").read() for r, _, fs in os.walk(d) for f in fs}


@pytest.mark.parametrize("flag,crit", [("--clean-scans", so.MAP), ("--clean-scans=scan-minus-map", so.SCAN_MINUS_MAP)])
def test_driver_clean_scans(tmp_path, small_pair, flag, crit):
    _dataset(tmp_path, small_pair)
    plain = _tree(_run(tmp_path, "plain", []))
    out = _run(tmp_path, "clean", [flag])
    clean = _tree(out)
    # without the flag nothing new is written; with it, the previous tree is unchanged and only the new files are added
    assert not any(k.startswith(("scan_static", "scan_dynamic")) for k in plain)
    assert {k: v for k, v in clean.items() if k in plain} == plain
    added = sorted(set(clean) - set(plain))
    assert all(k.startswith(("scan_static/", "scan_dynamic/", "map_static/", "map_dynamic/")) for k in added), added
    # the same run through the orchestrator, on the driver's keyframe selection and pose files: the files equal its scan sets
    c, q = small_pair
    kc = removert.parse_keyframes(c.K, 2, 5, 1)
    kq = removert.parse_keyframes_in_roi(q.poses, c.poses[kc], 1)
    G = removert.Removerter(num_knn=3, knn_thr=0.1)
    sel = []
    for s, d, ks in ((0, c, kc), (1, q, kq)):
        xyzi = np.concatenate([d.scan(k) for k in ks]); off = np.concatenate([[0], np.cumsum([len(d.scan(k)) for k in ks])])
        poses = removert.read_poses(str(tmp_path / ("central" if s == 0 else "query") / "poses.txt"))[ks]
        G.load_session_raw(s, xyzi, off, poses, removert.inverse_poses(poses))
        sel.append((list(ks), poses))
    G.run_step0()
    G.run_step12()
    G.run_step3()
    for s, name in ((0, "central"), (1, "query")):
        G.scanside_removal(s, s, crit)
        ks, poses = sel[s]
        for member, sub in (("scans_static_", "scan_static"), ("scans_dynamic_", "scan_dynamic")):
            exp = _per_kf(*G.scanset(member, s))
            files = sorted(os.listdir(out / sub / name))
            assert files == [f"{k:06d}.pcd" for k in ks]
            for fn, e in zip(files, exp):
                got = removert.read_pcd(str(out / sub / name / fn))
                assert got.shape == e.shape and np.array_equal(got.view(np.uint32), e.view(np.uint32)), (sub, name, fn)
        for member, sub, kind in (("scans_static_", "map_static", "Static"), ("scans_dynamic_", "map_dynamic", "Dynamic")):
            pts, off = G.scanset(member, s)
            glob = np.concatenate([so.local2global(pts[off[k]:off[k + 1]], poses[k]) for k in range(len(ks))])
            exp = oracle.voxel(glob, 0.05)
            got = removert.read_pcd(str(out / sub / f"{name.capitalize()}{kind}ScansMergedMapGlobal.pcd"))
            assert got.shape == exp.shape and np.array_equal(got.view(np.uint32), exp.view(np.uint32)), (sub, name)
    G.close()


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("split", [True, False])
def test_driver_clean_scans_two_ranks(tmp_path, small_pair, split):
    """Each rank splits its own keyframe block (session-split: its own session; otherwise a block of both) with no collective; the
    written tree equals the single-process one byte for byte."""
    _dataset(tmp_path, small_pair)
    args = ["--clean-scans=scan-minus-map"] + ([] if split else ["--no-split"])
    one = _tree(_run(tmp_path, "one", args))
    two = _tree(_run(tmp_path, "two", args, world=2))
    assert set(one) == set(two)
    for k in one:
        assert one[k] == two[k], k
