"""The ball subset of the map (ltr_remove_pass_ball) against the full map: `python profiles/map_ball_probe.py [config2|corridor] [K] [R]`.

config2: the configs[2]-shaped pair of bench.py (K keyframes per session, default 1000).  For each session's Step-0 map and each
    resolution (2.5, 2.375 = the revert's 0.95 r, 1.5) it runs one HD pass at fast_path 2 on the full map (ltr_remove_pass) and one on the
    balls of radius R (default the reference's kBallSize, 80 m), the two alternating, each after a warm-up pass that builds the kept scan
    images.  Per pass: the projection kernel's microseconds per launch (`ltr_profile_get`, the ball's tile-list kernel included), the
    share of pairs settled without exact arithmetic and the share skipped by whole tiles (`ltr_last_pass_stats` [1] / [0], [6] / [0]),
    and the flagged points per distance band from the nearest keyframe of the session.
corridor: n = 1, 2, 4, 8 copies of one session's lot, 250 m apart along x: the Step-0 map of K / n keyframes concatenated with its
    translated copies, and the same scans with translated poses.  Per n: the HD pass time per keyframe (`ltr_last_pass_stats` [4] / K)
    on the full map and on the balls, alternating.  Without the ball every launch visits every tile of the corridor.
The card name and power limit are read in the same run.  Nothing here is imported by the library or the tests."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BANDS = (0.0, 20.0, 40.0, 60.0, 80.0, np.inf)


def _card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return f"{torch.cuda.get_device_properties(0).name}; nvidia-smi: {q}"


def config2(kf, radius):
    import lt_mapper_b200 as ltr
    from lt_mapper_b200 import removert
    import bench
    from scipy.spatial import cKDTree
    print(f"# {_card()}; configs[2]-shaped pair, {kf} keyframes per session, R = {radius} m")
    blocks = bench.gen_block(0, kf)
    R = removert.Removerter(num_knn=bench.NUM_KNN, knn_thr=bench.KNN_THR, schedule=bench.SCHEDULE)
    for s, (d, inv) in enumerate(blocks):
        R.load_session(s, d.xyzi, d.offsets, d.poses, inv)
    R.run_step0()
    ctx = R.ctx
    rows = []
    for s in (0, 1):
        mh = R.cloud_handle("map_global_curr_", s)
        ss = R.scanset_handle("keyframe_scans_", s)
        pts = ctx.cloud_download(mh)
        dist, _ = cKDTree(blocks[s][0].poses[:, :3, 3]).query(pts[:, :3].astype(np.float64))
        band = np.digitize(dist, BANDS[1:-1])
        for a in (2.5, float(np.float32(0.95 * 2.5)), 1.5):
            runs = (("full", lambda: ctx.remove_pass(mh, ss, s, ltr.MODE_HD, a)),
                    (f"R = {radius:g}", lambda: ctx.remove_pass_ball(mh, ss, s, ltr.MODE_HD, a, radius)))
            for name, run in runs:
                run()                                            # warm: the kept scan images of this resolution
            for name, run in runs:
                ctx.profile_reset()
                n = run()
                st = ctx.last_pass_stats()
                pf = ctx.profile_get()
                flags = ctx.flags_download(mh).astype(bool)
                rows.append({"session": s, "alpha": a, "map": name, "map_points": len(pts), "flagged": int(n),
                             "kernel_us_per_launch": pf[0] / max(pf[1], 1.0), "launches": int(pf[1]), "pass_us": st[4],
                             "settled_fast": st[1] / st[0], "skipped_tiles": st[6] / st[0],
                             "flagged_per_band": [int((flags & (band == b)).sum()) for b in range(len(BANDS) - 1)]})
    R.close()
    print("| session | alpha | map | kernel us / launch | pass ms | settled fast [1]/[0] | whole tiles [6]/[0] | flagged 0-20 / 20-40 / 40-60 / 60-80 / >=80 m |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['session']} | {r['alpha']:.4g} | {r['map']} | {r['kernel_us_per_launch']:.0f} | {r['pass_us'] / 1e3:.1f} | "
              f"{100 * r['settled_fast']:.1f} % | {100 * r['skipped_tiles']:.1f} % | {' / '.join(map(str, r['flagged_per_band']))} |")
    print(json.dumps(rows))


def corridor(kf, radius):
    import lt_mapper_b200 as ltr
    import synth
    print(f"# {_card()}; corridor of n copies 250 m apart, {kf} keyframes in all, R = {radius:g} m")
    rows = []
    for n in (1, 2, 4, 8):
        k1 = kf // n
        d = synth.make_session(0, k1)
        inv = np.stack([np.linalg.inv(p) for p in d.poses])
        with ltr.Context() as ctx:
            ss1 = ctx.scanset_upload(d.xyzi, d.offsets)
            ps1 = ctx.poses_upload(d.poses, inv)
            m1 = ctx.cloud_download(ctx.voxel_centroid(ctx.merge_scans_global(ss1, ps1), 0.05))
            maps, poses = [], []
            for j in range(n):
                sh = np.array([250.0 * j, 0.0, 0.0], np.float32)
                mj = m1.copy()
                mj[:, :3] += sh
                maps.append(mj)
                pj = d.poses.copy()
                pj[:, :3, 3] += sh.astype(np.float64)
                poses.append(pj)
            P = np.concatenate(poses)
            xyzi = np.concatenate([d.xyzi] * n)
            off = np.concatenate([[0]] + [d.offsets[1:] + j * d.offsets[-1] for j in range(n)])
            mh = ctx.cloud_upload(np.concatenate(maps))
            ss = ctx.scanset_upload(xyzi, off)
            ps = ctx.poses_upload(P, np.stack([np.linalg.inv(p) for p in P]))
            K = len(P)
            runs = (("full", lambda: ctx.remove_pass(mh, ss, ps, ltr.MODE_HD, 2.5)),
                    (f"R = {radius:g}", lambda: ctx.remove_pass_ball(mh, ss, ps, ltr.MODE_HD, 2.5, radius)))
            for _, run in runs:
                run()
            for rep in range(2):
                for name, run in runs:
                    f = run()
                    st = ctx.last_pass_stats()
                    rows.append({"copies": n, "keyframes": K, "map_points": int(len(m1) * n), "map": name, "rep": rep, "flagged": int(f),
                                 "pass_us_per_kf": st[4] / K, "skipped_tiles": st[6] / st[0]})
    print("| copies | keyframes | map points | map | HD pass us / keyframe (two runs) | whole tiles [6]/[0] |")
    print("|---|---|---|---|---|---|")
    for i in range(0, len(rows), 4):
        for j in range(2):
            a, b = rows[i + j], rows[i + j + 2]
            print(f"| {a['copies']} | {a['keyframes']} | {a['map_points']} | {a['map']} | {a['pass_us_per_kf']:.0f}, {b['pass_us_per_kf']:.0f} | "
                  f"{100 * a['skipped_tiles']:.1f} % |")
    print(json.dumps(rows))


def main():
    part = sys.argv[1] if len(sys.argv) > 1 else "config2"
    kf = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
    radius = float(sys.argv[3]) if len(sys.argv) > 3 else 80.0
    sys.path.append(ROOT)
    {"config2": config2, "corridor": corridor}[part](kf, radius)


if __name__ == "__main__":
    main()
