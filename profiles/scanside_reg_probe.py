"""Scan-side removal between sessions with ICP fine registration (ltr_icp_refine_scanside + ltr_scanside_split_refined) on configs[2]-shaped
synthetic sessions (64 x 1800 scans, load-time VoxelGrid 0.05 m on the device) whose query poses carry a known error (0.3 m, 1 degree, in
the sensor frame).  Steps 0-2 run through the host orchestrator; then, for (map, scan) = (C,Q) and (Q,C), on the orchestrator's static
maps and full keyframe scans, it reports:
  * ltr_icp_refine_scanside's device time per keyframe against the other session's 0.4 m map (CUDA events on the context's stream),
  * ltr_scanside_split_refined's device time per keyframe, both criteria, against the full static map,
  * accepted keyframes (fitness < 1.0), the iteration histogram and exit reasons,
  * the dynamic point counts with and without registration (ltr_scanside_split on the same inputs).
Each timed call runs once untimed first; the minimum of two timed runs is reported.  A split's outputs are freed before the next call, so
every timed split draws its outputs from cached blocks, and the context's live bytes are the same before and after the measurements of a
session pair (checked).  With each split it reports ltr_scanside_stats (map / own-scan searches that reached the expanding pass).  Prints
one JSON object per session size; GPU name, power limit and SM clocks are read in the same run.
Usage: python profiles/scanside_reg_probe.py [keyframes_per_session ...]   (default: 100 1000)"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import synth  # noqa: E402
import oracle  # noqa: E402
import lt_mapper_b200 as ltr  # noqa: E402
from lt_mapper_b200 import removert  # noqa: E402

SIZES = [int(a) for a in sys.argv[1:]] or [100, 1000]


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


def timed(ctx, fn, release=None):
    """fn() once untimed, then the smaller of two CUDA-event timings (ms) and the last result.  release(out), when given, frees every
    result but the last one outside the timed window, before the next call: each timed call then draws its outputs from blocks the
    context's allocator already caches, as a steady-state caller's would, and nothing is left behind."""
    out = fn()
    best = None
    for _ in range(2):
        if release:
            release(out)
        ctx.synchronize()
        ctx.timer_start()
        out = fn()
        t = ctx.timer_stop()
        best = t if best is None else min(best, t)
    return best, out


def free_parts(ctx, pair):
    """Frees a (static, dynamic) pair of scan sets; returns their point counts."""
    n = [ctx.scanset_info(h)[1] for h in pair]
    for h in pair:
        ctx.scanset_free(h)
    return n


def probe(K):
    res = {"gpu": gpu_info(), "keyframes_per_session": K, "pose_error": "0.3 m, 1 deg (sensor frame, every query keyframe)"}
    sess = [synth.make_session(0, K), synth.make_session(1, K)]
    poses = [sess[0].poses, np.stack([p @ error_pose() for p in sess[1].poses])]
    G = removert.Removerter()
    for s in (0, 1):
        G.load_session_raw(s, sess[s].xyzi, sess[s].offsets, poses[s], oracle.inverse_poses(poses[s]))
    G.run_step0()
    G.run_step12()
    scans = [G.scanset("keyframe_scans_", s) for s in (0, 1)]
    maps = [G.cloud("map_global_curr_static_", s) for s in (0, 1)]
    G.close()
    del sess
    ctx = ltr.Context(device=0)
    for m_sess, s_sess, name in ((0, 1, "CQ"), (1, 0, "QC")):
        pts, off = scans[s_sess]
        ss = ctx.scanset_upload(pts, off)
        ps = ctx.poses_upload(poses[s_sess], oracle.inverse_poses(poses[s_sess]))
        mh = ctx.cloud_upload(maps[m_sess])
        td = ctx.voxel_centroid(mh, 0.4)
        ctx.synchronize()
        live0 = ctx.memory_stats()[0]
        t_icp, (T, fit, it, ex) = timed(ctx, lambda: ctx.icp_refine_scanside(ss, ps, td))
        acc = fit < 1.0
        r = {"scan_points": int(len(pts)), "map_points": int(len(maps[m_sess])), "target_points_0p4": int(ctx.cloud_size(td)),
             "icp_ms": t_icp, "icp_ms_per_keyframe": t_icp / K, "accepted": int(acc.sum()),
             "iteration_histogram": {int(v): int(n) for v, n in zip(*np.unique(it, return_counts=True))},
             "median_iterations": float(np.median(it)),
             "exit_reasons": {int(v): int(n) for v, n in zip(*np.unique(ex, return_counts=True))},
             "median_fitness": float(np.median(fit))}
        for crit, cname in ((ltr.SCANSIDE_MAP, "map"), (ltr.SCANSIDE_SCAN_MINUS_MAP, "scan_minus_map")):
            release = lambda pair: free_parts(ctx, pair)  # noqa: E731
            t_ref, parts = timed(ctx, lambda: ctx.scanside_split_refined(ss, ps, mh, crit, 2, 0.01, T, acc), release)
            st_ref = ctx.scanside_stats()
            n_ref = free_parts(ctx, parts)
            t_plain, parts = timed(ctx, lambda: ctx.scanside_split(ss, ps, mh, crit, 2, 0.01), release)
            st_plain = ctx.scanside_stats()
            n_plain = free_parts(ctx, parts)
            r[cname] = {"split_refined_ms_per_keyframe": t_ref / K, "split_plain_ms_per_keyframe": t_plain / K,
                        "dynamic_points_registered": int(n_ref[1]), "dynamic_points_unregistered": int(n_plain[1]),
                        "expanding_map_own_registered": [int(st_ref[1]), int(st_ref[2])],
                        "expanding_map_own_unregistered": [int(st_plain[1]), int(st_plain[2])]}
        res[name] = r
        assert ctx.memory_stats()[0] == live0, "a timed call left device memory behind"
        ctx.scanset_free(ss)
        ctx.poses_free(ps)
        ctx.cloud_free(mh)
        ctx.cloud_free(td)
    ctx.close()
    return res


def main():
    for K in SIZES:
        print(json.dumps(probe(K)), flush=True)


if __name__ == "__main__":
    main()
