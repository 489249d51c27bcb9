"""BASELINE configs[4] shape at single-GPU scale: an S-session cascaded LT-map.  Session 0 is the live map; every further session is
diffed against it (Steps 0-3) and the updated scans are promoted to the next live map (ltrh_cascade_promote_updated).  Wall-clock per
stage includes the pinned-host -> device upload of the new query session and the device-side VoxelGrid of the promoted scans (what the
reference's file protocol does at load).  Usage: python profiles/cascade_probe.py [sessions=6] [keyframes=100] > cascade.json"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import synth  # noqa: E402
from lt_mapper_b200 import removert  # noqa: E402

S = int(sys.argv[1]) if len(sys.argv) > 1 else 6
K = int(sys.argv[2]) if len(sys.argv) > 2 else 100
SCHEDULE = [(0, 2.5), (0, 2.0), (0, 1.5), (1, 1.0)]


def main():
    sess = [synth.make_session(s, K) for s in range(S)]
    inv = [np.stack([np.linalg.inv(p) for p in d.poses]) for d in sess]
    G = removert.Removerter(num_knn=1, knn_thr=0.04, schedule=SCHEDULE)
    G.load_session(0, sess[0].xyzi, sess[0].offsets, sess[0].poses, inv[0])
    stages = []
    t_all = time.perf_counter()
    for s in range(1, S):
        t0 = time.perf_counter()
        G.load_session(1, sess[s].xyzi, sess[s].offsets, sess[s].poses, inv[s])
        t1 = time.perf_counter()
        G.run_step0(); G.run_step12()
        t2 = time.perf_counter()
        G.run_step3()
        t3 = time.perf_counter()
        sizes = {n: int(G.cloud_size("saved:" + n)) for n in ("nd_map", "pd_map", "strong_nd_map", "strong_pd_map", "updated_map")}
        live = int(G.scanset("keyframe_scans_", 0)[1][-1])
        G.cascade_promote_updated()
        t4 = time.perf_counter()
        stages.append({"query_session": s, "upload_ms": (t1 - t0) * 1e3, "step0_12_ms": (t2 - t1) * 1e3, "step3_ms": (t3 - t2) * 1e3,
                       "promote_ms": (t4 - t3) * 1e3, "keyframes_per_s": 2 * K / (t4 - t0), "live_scan_points_in": live, **sizes})
    total = time.perf_counter() - t_all
    G.close()
    print(json.dumps({"workload": f"{S}-session cascade, {K} keyframes/session, 64x1800 scans, schedule {SCHEDULE}, kNN k=1 thr=0.04, 1x H100",
                      "total_s": total, "keyframes_per_s_overall": 2 * K * (S - 1) / total, "stages": stages}, indent=1))


if __name__ == "__main__":
    main()
