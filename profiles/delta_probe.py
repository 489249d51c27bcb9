"""LT-map change composition and map rollback (DESIGN.md §5.3) on a BASELINE configs[2]-shaped cascade: sessions 0..T of synth at K
keyframes (64 x 1800 scans, loaded through the load-time VoxelGrid 0.05 as the driver loads them; schedule [(0, 2.5), (0, 2.0), (0, 1.5),
(1, 1.0)], kNN k = 1, thr = 0.04) promoted T times with delta maps on, then compose_changes(0, T) and rollback(0) timed with CUDA events on the context's stream, the primitive ltr_knn_split_per_keyframe
(live scans against the composed PD) per keyframe, the delta sizes against the live scans, and the CPU restatement
(tests/_delta_oracle.py) on one sampled keyframe.  Usage: python profiles/delta_probe.py [generations=3] [keyframes=100 ...] > delta.json"""
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
import _delta_oracle as D  # noqa: E402
from lt_mapper_b200 import removert  # noqa: E402

T = int(sys.argv[1]) if len(sys.argv) > 1 else 3
KS = [int(a) for a in sys.argv[2:]] or [100, 1000]
SCHEDULE = [(0, 2.5), (0, 2.0), (0, 1.5), (1, 1.0)]
KNN, THR = 1, 0.04


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:   # the number is still reported, without the card
        return f"unknown ({e})"


def timed(G, fn, reps=3):
    fn()                     # warm-up: module load, allocator
    ms = []
    for _ in range(reps):
        G.ctx.timer_start()
        fn()
        ms.append(G.ctx.timer_stop())
    return float(np.median(ms))


def run(K):
    G = removert.Removerter(num_knn=KNN, knn_thr=THR, schedule=SCHEDULE)
    G.set_delta_maps(True)
    s0 = synth.make_session(0, K)
    G.load_session_raw(0, s0.xyzi, s0.offsets, s0.poses, removert.inverse_poses(s0.poses))
    del s0
    gens = []
    for s in range(1, T + 1):
        q = synth.make_session(s, K)
        G.load_session_raw(1, q.xyzi, q.offsets, q.poses, removert.inverse_poses(q.poses))
        del q
        G.run_step0(); G.run_step12(); G.run_step3()
        live = G.ctx.scanset_info(G.scanset_handle("keyframe_scans_", 0))[1]
        pd = G.ctx.scanset_info(G.scanset_handle("keyframe_scans_pd_", 0))[1]
        nd = G.ctx.scanset_info(G.scanset_handle("keyframe_scans_strong_nd_", 0))[1]
        gens.append({"generation": s - 1, "live_points": live, "pd_points": pd, "nd_points": nd, "pd_share": pd / live, "nd_share": nd / live})
        G.cascade_promote_updated()
    live = G.ctx.scanset_info(G.scanset_handle("keyframe_scans_", 0))[1]
    compose_ms = timed(G, lambda: G.compose_changes(0, T))
    rollback_ms = timed(G, lambda: G.rollback(0))
    pd_h = G.scanset_handle("composed_pd_", 0)
    live_h = G.scanset_handle("keyframe_scans_", 0)

    def prim():
        n, f = G.ctx.knn_split_per_keyframe(live_h, pd_h, KNN, THR)
        G.ctx.scanset_free(n); G.ctx.scanset_free(f)
    prim_ms = timed(G, prim)
    # the CPU restatement of rollback(0) on one sampled keyframe
    k = K // 2
    live_k = D.split_sets(*G.scanset("keyframe_scans_", 0))[k]
    deltas = []
    for g in range(T):
        G.compose_changes(g, g + 1)
        deltas.append(([D.split_sets(*G.scanset("composed_pd_", 0))[k]], [D.split_sets(*G.scanset("composed_nd_", 0))[k]]))
    t0 = time.perf_counter()
    D.rollback([live_k], deltas, 0, KNN, THR)
    oracle_s = time.perf_counter() - t0
    restored = G.ctx.scanset_info(G.scanset_handle("keyframe_scans_restored_", 0))[1]
    G.close()
    return {"keyframes": K, "generations": gens, "live_points": live, "restored_points": restored,
            "compose_changes_ms": compose_ms, "compose_changes_ms_per_keyframe": compose_ms / K,
            "rollback_ms": rollback_ms, "rollback_ms_per_keyframe": rollback_ms / K,
            "knn_split_per_keyframe_ms": prim_ms, "knn_split_per_keyframe_us_per_keyframe": prim_ms * 1e3 / K,
            "oracle_rollback_one_keyframe_s": oracle_s}


def main():
    out = {"workload": f"{T}-generation cascade, 64x1800 scans after the load-time VoxelGrid 0.05, schedule {SCHEDULE}, kNN k={KNN} thr={THR}", "card": card(),
           "runs": [run(K) for K in KS]}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
