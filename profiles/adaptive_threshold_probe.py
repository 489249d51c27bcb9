"""The range-adaptive threshold against the constant 0.1 m on the configs[2] maps: `python profiles/adaptive_threshold_probe.py [KF] [c]`.

For each session's Step-0 map and each resolution of the selfRemovert schedule (r and the revert's 0.95 r) it runs one HD pass at
fast_path 2 with the constant threshold (ltr_remove_pass) and one with fl(c * scan range) (ltr_remove_pass_adaptive, c = 0.05 by
default), and prints per pass: the projection kernel's microseconds per launch (`ltr_profile_get`), the culled share and the pairs
through the exact-range and the full exact paths (`ltr_last_pass_stats` [6], [2], [5]), and the flagged points per range band.  A
flagged point's band is its distance from the nearest keyframe origin of the session, which stands in for the scan range it was
compared with.  The card name and power limit are read in the same run.  Nothing here is imported by the library or the tests."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BANDS = (0.0, 20.0, 40.0, 60.0, np.inf)


def main():
    kf = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
    coeff = float(sys.argv[2]) if len(sys.argv) > 2 else 0.05
    sys.path.append(ROOT)
    import lt_mapper_b200 as ltr
    from lt_mapper_b200 import removert
    import bench
    from scipy.spatial import cKDTree
    import torch
    p = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# {p.name}; nvidia-smi: {q}; {kf} keyframes per session, c = {coeff}")
    blocks = bench.gen_block(0, kf)
    R = removert.Removerter(num_knn=bench.NUM_KNN, knn_thr=bench.KNN_THR, schedule=bench.SCHEDULE)
    for s, (d, inv) in enumerate(blocks):
        R.load_session(s, d.xyzi, d.offsets, d.poses, inv)
    R.run_step0()
    ctx = R.ctx
    alphas = []
    for r in bench.RESOLUTIONS:
        alphas += [r, float(np.float32(0.95 * r))]
    rows = []
    for s in (0, 1):
        mh = R.cloud_handle("map_global_curr_", s)
        ss = R.scanset_handle("keyframe_scans_", s)
        pts = ctx.cloud_download(mh)
        dist, _ = cKDTree(blocks[s][0].poses[:, :3, 3]).query(pts[:, :3].astype(np.float64))
        band = np.digitize(dist, BANDS[1:-1])
        for a in alphas:
            for name, run in (("0.1 m", lambda: ctx.remove_pass(mh, ss, s, ltr.MODE_HD, a)),
                              (f"{coeff} s", lambda: ctx.remove_pass_adaptive(mh, ss, s, ltr.MODE_HD, a, coeff))):
                run()                                            # warm: the kept scan images of this resolution
                ctx.profile_reset()
                n = run()
                st = ctx.last_pass_stats()
                pf = ctx.profile_get()
                flags = ctx.flags_download(mh).astype(bool)
                per_band = [int((flags & (band == b)).sum()) for b in range(len(BANDS) - 1)]
                rows.append({"session": s, "alpha": a, "threshold": name, "map_points": len(pts), "flagged": int(n),
                             "kernel_us_per_launch": pf[0] / max(pf[1], 1.0), "launches": int(pf[1]), "culled": st[6] / st[0],
                             "exact_range_pairs": int(st[2] - st[5]), "exact_full_pairs": int(st[5]), "flagged_per_band": per_band})
    R.close()
    print("| session | alpha | threshold | kernel us / launch | culled | exact-range pairs | full exact pairs | flagged 0-20 / 20-40 / 40-60 / >=60 m |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['session']} | {r['alpha']:.4g} | {r['threshold']} | {r['kernel_us_per_launch']:.1f} | {100 * r['culled']:.1f} % | "
              f"{r['exact_range_pairs']} | {r['exact_full_pairs']} | {' / '.join(map(str, r['flagged_per_band']))} |")
    print(json.dumps(rows))


if __name__ == "__main__":
    main()
