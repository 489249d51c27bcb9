"""ICP refinement of the low-dynamic kNN diff (icp.cu) on configs[2]-shaped synthetic sessions (64 x 1800 scans, load-time VoxelGrid
0.05 m on the device) whose query poses carry a known error (0.3 m, 1 degree, in the sensor frame).  Runs Steps 0-2 through the host
orchestrator with the refinement off and on and reports:
  * the 0.4 m source sizes (a sample of query keyframes, voxelised by the CPU oracle) and the 0.4 m target size,
  * the iteration histogram, exit reasons and accepted share of both sessions,
  * ltr_icp_refine's device time per keyframe (CUDA events on the context's stream, query keyframes against the central map),
  * the added Step 2 time (the orchestrator's "ld_knn" stage, on minus off; host clock around synchronised calls),
  * the CPU restatement's (tests/_icp_oracle.py) time for one keyframe, and whether it equals the device bit for bit.
Prints one JSON object; GPU name, power limit and SM clocks are read in the same run.
Usage: python profiles/icp_probe.py [keyframes_per_session=100]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth  # noqa: E402
import oracle  # noqa: E402
import lt_mapper_b200 as ltr  # noqa: E402
from lt_mapper_b200 import removert  # noqa: E402
import _icp_oracle as io  # noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 else 100
SAMPLE = 8


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def error_pose():
    a, b = np.deg2rad(1.0), np.deg2rad(1.0 / 3)
    Rz = np.array([[np.cos(a), -np.sin(a), 0, 0], [np.sin(a), np.cos(a), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    Rx = np.array([[1, 0, 0, 0], [0, np.cos(b), -np.sin(b), 0], [0, np.sin(b), np.cos(b), 0], [0, 0, 0, 1]])
    E = Rz @ Rx
    E[:3, 3] = np.array([1.0, -0.6, 0.2]) * 0.3
    return E


def main():
    res = {"gpu": gpu_info(), "keyframes_per_session": K, "pose_error": "0.3 m, 1 deg (sensor frame, every query keyframe)"}
    c, q = synth.make_session(0, K), synth.make_session(1, K)
    qp = np.stack([p @ error_pose() for p in q.poses])
    runs = {}
    for on in (False, True):
        G = removert.Removerter()
        G.set_icp_refinement(on)
        G.load_session_raw(0, c.xyzi, c.offsets, c.poses, oracle.inverse_poses(c.poses))
        G.load_session_raw(1, q.xyzi, q.offsets, qp, oracle.inverse_poses(qp))
        G.run_step0()
        G.run_step12()
        runs[on] = {"ld_knn_ms": 1e3 * G.timing("ld_knn"), "nd_pd_candidates": [G.ctx.scanset_info(G.scanset_handle("scans_knn_diff_", s))[1] for s in (0, 1)]}
        if on:
            for s, name in ((0, "central"), (1, "query")):
                st = G.icp_stats(s)
                runs[on][name] = {"iteration_histogram": {int(v): int(n) for v, n in zip(*np.unique(st["iterations"], return_counts=True))},
                                  "exit_reasons": {int(v): int(n) for v, n in zip(*np.unique(st["exit"], return_counts=True))},
                                  "accepted": int(st["accepted"].sum()), "median_fitness": float(np.median(st["fitness"]))}
            scans, off = G.scanset("keyframe_scans_static_projected_", 1)
            cmap = G.cloud("map_global_curr_static_", 0)
        G.close()
    res["added_step2_ms"] = runs[True]["ld_knn_ms"] - runs[False]["ld_knn_ms"]
    res["runs"] = {"off": runs[False], "on": runs[True]}
    # device time of ltr_icp_refine alone: query keyframes against the central map
    ctx = ltr.Context(device=0)
    ss = ctx.scanset_upload(scans, off)
    ps = ctx.poses_upload(qp, oracle.inverse_poses(qp))
    th = ctx.cloud_upload(cmap)
    td = ctx.voxel_centroid(th, 0.4)
    md = ctx.cloud_download(td)
    res["static_projected_points_per_keyframe"] = float(np.diff(off).mean())
    res["target_points_0p4"] = int(len(md))
    times = []
    for r in range(3):
        ctx.synchronize()
        ctx.timer_start()
        T, fit, it, ex = ctx.icp_refine(ss, ps, td)
        times.append(ctx.timer_stop())
    res["icp_refine_ms"] = times
    res["icp_ms_per_keyframe"] = min(times) / K
    sample = np.linspace(0, K - 1, SAMPLE).astype(int)
    sizes = [len(oracle.voxel(io.global_scan(scans[off[k]:off[k + 1]], qp[k]), 0.4)) for k in sample]
    res["source_points_0p4_sample"] = {"min": int(min(sizes)), "median": float(np.median(sizes)), "max": int(max(sizes))}
    k = int(sample[len(sample) // 2])
    t0 = time.perf_counter()
    eT, efit, eit, eex = io.refine_session(scans[off[k]:off[k + 1]], np.array([0, off[k + 1] - off[k]]), qp[k:k + 1], md)
    res["restatement_s_one_keyframe"] = time.perf_counter() - t0
    res["restatement_equals_device"] = bool(np.array_equal(eT[0].view(np.uint32), T[k].view(np.uint32)) and efit[0] == fit[k] and
                                            eit[0] == it[k] and eex[0] == ex[k])
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
