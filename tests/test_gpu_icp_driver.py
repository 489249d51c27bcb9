"""The drop-in driver's --icp-refinement: the output tree keeps its layout, the saved maps equal what the orchestrator holds with
Removerter.set_icp_refinement(True), the summary line reports the orchestrator's accepted count and median iterations, and a 2-rank run
writes the single-process tree when two GPUs are visible."""
import os
import re
import subprocess

import numpy as np
import pytest

from lt_mapper_b200 import removert
from test_gpu_scanside_orchestrator import BIN, _PARAMS, _dataset, _n_gpus, _tree

pytestmark = pytest.mark.gpu
SUMMARY = re.compile(r" ICP refinement: (\d+) of (\d+) keyframes accepted, median iterations (\d+)")


def _run(tmp_path, tag, args, world=1):
    out = tmp_path / f"out_{tag}"
    cfg = tmp_path / f"params_{tag}.yaml"
    cfg.write_text(_PARAMS.format(out=out, d=tmp_path))
    outputs = []
    if world == 1:
        r = subprocess.run([BIN, "--config", str(cfg)] + args, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        outputs.append(r.stdout)
    else:
        procs = []
        for rank in range(world):
            e = dict(os.environ, RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), LTR_NCCL_ID_FILE=str(tmp_path / f"nccl_{tag}"))
            procs.append(subprocess.Popen([BIN, "--config", str(cfg)] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=e))
        for p in procs:
            o, _ = p.communicate(timeout=600)
            assert p.returncode == 0, o
            outputs.append(o)
    return out, "".join(outputs)


def test_driver_icp_refinement_writes_what_the_orchestrator_holds(tmp_path, small_pair):
    _dataset(tmp_path, small_pair)
    out_plain, log_plain = _run(tmp_path, "plain", [])
    out, log = _run(tmp_path, "icp", ["--icp-refinement"])
    plain, icp = _tree(out_plain), _tree(out)
    assert set(plain) == set(icp), "the option must not change the output tree's layout"
    assert not SUMMARY.search(log_plain)
    m = SUMMARY.search(log)
    assert m, log
    # the same run through the orchestrator, on the driver's keyframe selection and pose files
    c, q = small_pair
    kc = removert.parse_keyframes(c.K, 2, 5, 1)
    kq = removert.parse_keyframes_in_roi(q.poses, c.poses[kc], 1)
    G = removert.Removerter(num_knn=3, knn_thr=0.1)
    G.set_icp_refinement(True)
    for s, d, ks in ((0, c, kc), (1, q, kq)):
        xyzi = np.concatenate([d.scan(k) for k in ks])
        off = np.concatenate([[0], np.cumsum([len(d.scan(k)) for k in ks])])
        poses = removert.read_poses(str(tmp_path / ("central" if s == 0 else "query") / "poses.txt"))[ks]
        G.load_session_raw(s, xyzi, off, poses, removert.inverse_poses(poses))
    G.run_step0()
    G.run_step12()
    st = [G.icp_stats(s) for s in (0, 1)]
    its = np.sort(np.concatenate([x["iterations"] for x in st]))
    assert int(m.group(1)) == sum(int(x["accepted"].sum()) for x in st) and int(m.group(2)) == len(its)
    assert int(m.group(3)) == int(its[(len(its) - 1) // 2])
    G.run_step3()
    compared = []
    for rel, data in icp.items():
        if "/" in rel or not rel.endswith(".pcd"):
            continue
        try:
            exp = G.cloud("saved:" + rel[:-4])
        except Exception:  # noqa: BLE001 -- files that are not saved maps of the orchestrator
            continue
        got = removert.read_pcd(str(out / rel))
        assert got.shape == exp.shape and np.array_equal(got.view(np.uint32), exp.view(np.uint32)), rel
        compared.append(rel)
    assert {"nd_map.pcd", "pd_map.pcd"} <= set(compared), compared
    assert icp["nd_map.pcd"] != plain["nd_map.pcd"] or icp["pd_map.pcd"] != plain["pd_map.pcd"], "the refinement changed nothing"
    G.close()


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("split", [True, False])
def test_driver_icp_refinement_two_ranks(tmp_path, small_pair, split):
    """Each rank refines its own keyframe block against its replica of the other map, with no collective: the tree and the summary line
    equal the single-process run."""
    _dataset(tmp_path, small_pair)
    args = ["--icp-refinement"] + ([] if split else ["--no-split"])
    out1, log1 = _run(tmp_path, "one", args)
    out2, log2 = _run(tmp_path, "two", args, world=2)
    assert SUMMARY.search(log1).groups() == SUMMARY.search(log2).groups()
    one, two = _tree(out1), _tree(out2)
    assert set(one) == set(two)
    for k in one:
        assert one[k] == two[k], k
