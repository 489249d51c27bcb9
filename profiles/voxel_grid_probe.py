"""Load-time VoxelGrid: host restatement (removert.voxel_grid_scans, io.cpp on OpenMP threads) against the device entry
(ltr_voxel_grid_per_keyframe) on configs[2]-shaped synthetic sessions (64 x 1800 scans), at leaves 0.05 and 0.2.  Also times what a
cascade promotion of such a session costs both ways: the old round trip (download, host filter, upload) against the device filter.
Every device output is compared bit for bit with the host one.  Prints one JSON object; GPU name, power limit and SM clocks are read
in the same run.  Usage: python profiles/voxel_grid_probe.py [keyframes_per_session=1000] [sessions=2]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import synth  # noqa: E402
import lt_mapper_b200 as ltr  # noqa: E402
from lt_mapper_b200 import removert  # noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
S = int(sys.argv[2]) if len(sys.argv) > 2 else 2
REPS = 3


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def main():
    res = {"keyframes_per_session": K, "sessions": S, "omp_threads": os.environ.get("OMP_NUM_THREADS", str(os.cpu_count())), "runs": []}
    ctx = ltr.Context(device=0)
    for s in range(S):
        d = synth.make_session(s, K)
        for leaf in (0.05, 0.2):
            t0 = time.perf_counter()
            exp, exp_off = removert.voxel_grid_scans(d.xyzi, d.offsets, leaf)
            host_ms = (time.perf_counter() - t0) * 1e3
            n_ov = int(np.sum([(exp_off[k + 1] - exp_off[k]) == (d.offsets[k + 1] - d.offsets[k]) for k in range(K)]))
            h = ctx.scanset_upload(d.xyzi, d.offsets)
            o, nov = ctx.voxel_grid_per_keyframe(h, leaf)      # warm-up (module load, allocator)
            ctx.scanset_free(o)
            dev_ms = []
            for _ in range(REPS):
                ctx.synchronize()
                ctx.timer_start()
                o, nov = ctx.voxel_grid_per_keyframe(h, leaf)
                dev_ms.append(ctx.timer_stop())
                ctx.scanset_free(o)
            o, nov = ctx.voxel_grid_per_keyframe(h, leaf)
            got, got_off = ctx.scanset_download(o)
            ctx.scanset_free(o)
            equal = bool(np.array_equal(got_off, exp_off) and np.array_equal(got.view(np.uint32), exp.view(np.uint32)))
            # the promotion before this change: download the live scans, filter them on the host, upload the result
            t0 = time.perf_counter()
            x, off = ctx.scanset_download(h)
            y, yo = removert.voxel_grid_scans(x, off, leaf)
            u = ctx.scanset_upload(y, yo)
            ctx.synchronize()
            roundtrip_ms = (time.perf_counter() - t0) * 1e3
            ctx.scanset_free(u)
            t0 = time.perf_counter()
            o, _ = ctx.voxel_grid_per_keyframe(h, leaf)
            ctx.synchronize()
            device_promote_ms = (time.perf_counter() - t0) * 1e3
            ctx.scanset_free(o)
            ctx.scanset_free(h)
            res["runs"].append({"session": s, "leaf": leaf, "points": int(d.offsets[-1]), "host_overflow_exits": n_ov, "device_overflow_exits": nov,
                                "host_filter_ms": host_ms, "device_filter_ms": float(np.median(dev_ms)), "device_filter_ms_all": dev_ms,
                                "promote_roundtrip_ms": roundtrip_ms, "promote_device_ms": device_promote_ms, "bit_equal": equal})
    res["gpu"] = gpu_info()
    ctx.close()
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
