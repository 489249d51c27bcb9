"""Multi-GPU parity of LT-map change composition and map rollback (DESIGN.md §5.3): when the box has >= 2 GPUs, 2 ranks over NCCL, session
split and not, record, compose and restore their own central keyframes, and every composed / restored cloud and the restored map must
equal the single-process run byte for byte.  The same for the driver's --compose started once per GPU."""
import filecmp
import glob
import json
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _run(n, out, split):
    worker = os.path.join(ROOT, "tests", "_delta_rank_worker.py")
    args = ["--out", out, "--kf", "6", "--split", str(split)]
    if n == 1:
        cmd = [sys.executable, worker] + args
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
               "--master-port", str(29700 + 7 * n + split), worker] + args
    env = dict(os.environ, LTR_DIST_VOXEL_MIN="1000")   # the restored map goes through the distributed voxeliser too
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    merged = {}
    for f in sorted(glob.glob(os.path.join(out, "rank*.json"))):
        for k, v in json.load(open(f)).items():
            assert merged.setdefault(k, v) == v, f"replicas disagree on {k}"
    return merged


@pytest.mark.parametrize("split", [1, 0])
def test_delta_maps_two_ranks_equal_one_rank(tmp_path, split):
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    one = _run(1, str(tmp_path / "one"), 0)
    two = _run(2, str(tmp_path / f"two{split}"), split)
    assert one["delta_count"] == 2 and len(one) > 6 * 9
    assert sorted(one) == sorted(two), sorted(set(one) ^ set(two))[:10]
    bad = [k for k in one if two[k] != one[k]]
    assert not bad, bad[:10]


def test_driver_compose_on_two_gpus_writes_the_single_process_tree(tmp_path):
    """Two cascade generations through the single-process driver, then --compose once in one process and once per GPU (split and
    --no-split): the composed tree is the same file for file.  A delta file missing from the second rank's block stops both ranks."""
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    import synth
    from lt_mapper_b200 import removert
    from test_gpu_driver import BIN, _write_session
    K = 6
    for name, s in zip("abc", [synth.make_session(s, K, beams=32, az_steps=900) for s in (0, 1, 2)]):
        _write_session(tmp_path / name, s)

    def cfg(central, query, out):
        p = tmp_path / f"params_{out}.yaml"
        p.write_text("removert:\n  saveMapPCD: true\n" + f'  save_pcd_directory: "{tmp_path / out}"\n'
                     + f'  central_sess_scan_dir: "{central}"\n  central_sess_pose_path: "{tmp_path}/a/poses.txt"\n'
                     + f'  query_sess_scan_dir: "{tmp_path}/{query}/Scans/"\n  query_sess_pose_path: "{tmp_path}/{query}/poses.txt"\n'
                     + "  sequence_vfov: 50\n  sequence_hfov: 360\n  keyframe_gap: 1\n  start_idx: 0\n  end_idx: 100\n"
                     + "  downsample_voxel_size: 0.05\n  num_nn_points_within: 2\n  dist_nn_points_within: 0.01\n")
        return str(p)

    for central, query, out in ((tmp_path / "a" / "Scans", "b", "out1"), (tmp_path / "central2", "c", "out2")):
        r = subprocess.run([BIN, "--config", cfg(central, query, out)], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        shutil.copytree(tmp_path / out / "scans_updated", tmp_path / ("central2" if out == "out1" else "central3"))
    compose = f"--compose={tmp_path}/out1,{tmp_path}/out2"
    r = subprocess.run([BIN, "--config", cfg(tmp_path / "central3", "c", "one"), compose], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr

    def two(mode, extra):
        procs = []
        for rank in range(2):
            env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank), MASTER_PORT="29611", LTR_NCCL_ID_FILE=str(tmp_path / f"id_{mode}"),
                       LTR_DIST_VOXEL_MIN="1000")
            procs.append(subprocess.Popen([BIN, "--config", cfg(tmp_path / "central3", "c", mode), compose] + extra, env=env, stdout=subprocess.PIPE,
                                          stderr=subprocess.STDOUT, text=True))
        outs = [p.communicate(timeout=600)[0] for p in procs]
        return [p.returncode for p in procs], "\n".join(outs)

    def tree(d):
        return sorted(os.path.relpath(os.path.join(p, f), d) for p, _, fs in os.walk(d) for f in fs)
    files = tree(tmp_path / "one")
    nk = len(removert.parse_keyframes(K, 0, 100, 1))
    assert nk >= 2 and len(files) == 3 * nk + 1 and "composed/restored_map.pcd" in files, files
    for mode, extra in (("two_split", []), ("two_blocks", ["--no-split"])):
        rcs, log = two(mode, extra)
        assert rcs == [0, 0], log
        assert tree(tmp_path / mode) == files, mode
        for f in files:
            assert filecmp.cmp(tmp_path / "one" / f, tmp_path / mode / f, shallow=False), (mode, f)
    last = sorted(os.listdir(tmp_path / "out2" / "scans_nd_strong"))[-1]     # in the second rank's block with --no-split
    os.remove(tmp_path / "out2" / "scans_nd_strong" / last)
    rcs, log = two("two_missing", ["--no-split"])
    assert rcs[0] != 0 and rcs[1] != 0 and last in log, log
