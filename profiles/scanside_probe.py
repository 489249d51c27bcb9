"""Scan-side removal (ltr_scanside_split) on configs[2]-shaped synthetic sessions (64 x 1800 scans, load-time VoxelGrid 0.05 m on the
device, maps = 0.05 m octree centroids of the merged scans): per criterion and (map, scan) pair, device time per keyframe, points per
second and the share of searches that reached the expanding pass; beside it the CPU oracle's time (tests/_scanside_oracle.py, one
thread of k-d tree queries) on one sampled keyframe, compared bit for bit with the device.  Prints one JSON object; GPU name, power limit
and SM clocks are read in the same run.  Usage: python profiles/scanside_probe.py [keyframes_per_session=200] [k=3] [thr=0.1]"""
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
import _scanside_oracle as so  # noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 else 200
KNN = int(sys.argv[2]) if len(sys.argv) > 2 else 3
THR = float(sys.argv[3]) if len(sys.argv) > 3 else 0.1
REPS = 3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def main():
    res = {"gpu": gpu_info(), "keyframes_per_session": K, "k": KNN, "thr": THR, "runs": []}
    ctx = ltr.Context(device=0)
    sess = []
    for s in range(2):
        d = synth.make_session(s, K)
        raw = ctx.scanset_upload(d.xyzi, d.offsets)
        vg, _ = ctx.voxel_grid_per_keyframe(raw, 0.05)
        ctx.scanset_free(raw)
        inv = np.stack([oracle.inverse4x4(p) for p in d.poses])
        ps = ctx.poses_upload(d.poses, inv)
        merged = ctx.merge_scans_global(vg, ps)
        mh = ctx.voxel_centroid(merged, 0.05)
        ctx.cloud_free(merged)
        sess.append((vg, ps, mh, d.poses, inv))
    res["scan_points"] = [ctx.scanset_info(s[0])[1] for s in sess]
    res["map_points"] = [ctx.cloud_size(s[2]) for s in sess]
    for crit_name, crit in (("map", so.MAP), ("scan_minus_map", so.SCAN_MINUS_MAP)):
        for pair in ("CC", "QQ", "CQ", "QC"):
            m, s = sess["CQ".index(pair[0])], sess["CQ".index(pair[1])]
            npts = ctx.scanset_info(s[0])[1]
            times = []
            for r in range(REPS + 1):
                ctx.synchronize()
                t0 = time.perf_counter()
                st, dy = ctx.scanside_split(s[0], s[1], m[2], crit, KNN, THR)
                ctx.synchronize()
                dt = time.perf_counter() - t0
                if r > 0:
                    times.append(dt)
                stats = ctx.scanside_stats()
                if r < REPS:
                    ctx.scanset_free(st)
                    ctx.scanset_free(dy)
            t = float(np.median(times))
            run = {"criterion": crit_name, "pair": pair, "seconds": t, "ms_per_keyframe": 1e3 * t / K, "points_per_second": npts / t,
                   "expanding_share_map": float(stats[1]) / max(npts, 1), "expanding_share_scan": float(stats[2]) / max(npts, 1),
                   "launches": int(stats[3])}
            if pair in ("CC", "QC"):
                # the oracle on one sampled keyframe, checked bit for bit
                kf = K // 2
                pts, off = ctx.scanset_download(s[0])
                mp = ctx.cloud_download(m[2])
                t0 = time.perf_counter()
                e_st, e_dy, _ = so.split_scan(pts[off[kf]:off[kf + 1]], s[3][kf], s[4][kf], mp, crit, KNN, THR)
                run["oracle_seconds_one_keyframe"] = time.perf_counter() - t0
                d_st, o_st = ctx.scanset_download(st)
                d_dy, o_dy = ctx.scanset_download(dy)
                run["oracle_match"] = bool(np.array_equal(d_st[o_st[kf]:o_st[kf + 1]].view(np.uint32), e_st.view(np.uint32)) and
                                           np.array_equal(d_dy[o_dy[kf]:o_dy[kf + 1]].view(np.uint32), e_dy.view(np.uint32)))
                run["static_share"] = float(o_st[-1]) / max(npts, 1)
            ctx.scanset_free(st)
            ctx.scanset_free(dy)
            res["runs"].append(run)
            print(json.dumps(run), file=sys.stderr, flush=True)
    res["memory_live_cached_peak"] = ctx.memory_stats()
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
