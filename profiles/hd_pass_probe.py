"""Per-pass figures of the scan-minus-map projection (HD remove / revert) on the configs[2] maps: `python profiles/hd_pass_probe.py [KF] [--no-diag]`.

For each session's Step-0 map and each resolution of the selfRemovert schedule (r and the revert's 0.95 r) it runs one HD pass at
fast_path 2 and prints, per pass: (point, keyframe) pairs, the culled share (`ltr_last_pass_stats` [6]), the exact-path shares ([2], [5])
and the projection kernel's microseconds per launch (`ltr_profile_get`).  It then builds a diagnostic copy of the CUDA library with
-DLTR_PROBE_NOMAYBE in a temporary directory and repeats the passes there: that build reports, in place of the atomics count, the
non-culled (128-point tile, keyframe) iterations in which no lane took the `maybe` branch, i.e. the pairs any tile-level cull could still
remove.  The diagnostic build is slower; its times are not reported.  Nothing here is imported by the library or the tests."""
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_passes(kf):
    sys.path.append(ROOT)     # after PYTHONPATH: the diagnostic child imports the package from its temporary copy
    import lt_mapper_b200 as ltr
    from lt_mapper_b200 import removert
    import bench              # puts ROOT first on sys.path: import the package before it
    assert os.environ.get("LTR_PROBE_CHILD") != "1" or not ltr.__file__.startswith(ROOT), ltr.__file__
    blocks = bench.gen_block(0, kf)
    R = removert.Removerter(num_knn=bench.NUM_KNN, knn_thr=bench.KNN_THR, schedule=bench.SCHEDULE)
    for s, (d, inv) in enumerate(blocks):
        R.load_session(s, d.xyzi, d.offsets, d.poses, inv)
    R.run_step0()
    ctx = R.ctx
    alphas = []
    for r in bench.RESOLUTIONS:
        alphas += [r, float(__import__("numpy").float32(0.95 * r))]
    out = []
    for s in (0, 1):
        mh = R.cloud_handle("map_global_curr_", s)
        ss = R.scanset_handle("keyframe_scans_", s)
        n = ctx.cloud_size(mh)
        for a in alphas:
            ctx.remove_pass(mh, ss, s, ltr.MODE_HD, a)        # warm
            ctx.profile_reset()
            nd = ctx.remove_pass(mh, ss, s, ltr.MODE_HD, a)
            st = ctx.last_pass_stats()
            pf = ctx.profile_get()
            out.append({"session": s, "alpha": a, "map_points": n, "flagged": int(nd), "pairs": st[0], "culled": st[6] / st[0],
                        "exact": st[2] / st[0], "exact_full": st[5] / st[0], "counter1": st[3], "pass_ms": st[4] / 1e3,
                        "kernel_us_per_launch": pf[0] / max(pf[1], 1.0), "launches": int(pf[1])})
    R.close()
    return out


def main():
    kf = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 1000
    if os.environ.get("LTR_PROBE_CHILD") == "1":
        print(json.dumps(run_passes(kf)))
        return
    import torch
    p = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# {p.name}; nvidia-smi: {q}")
    normal = run_passes(kf)
    if "--no-diag" in sys.argv:
        print(json.dumps({"normal": normal}))
        for a in normal:
            print(f"| {a['session']} | {a['alpha']:.3f} | {a['culled']:.4f} | {a['exact']:.4f} | {a['exact_full']:.5f} | {a['kernel_us_per_launch']:.0f} | {a['pass_ms']:.1f} |")
        return
    tmp = tempfile.mkdtemp(prefix="ltr_probe_")
    try:
        shutil.copytree(os.path.join(ROOT, "lt_mapper_b200"), os.path.join(tmp, "lt_mapper_b200"),
                        ignore=shutil.ignore_patterns("*.o", "*.so", "*.ptxas.log", "__pycache__", "ltremovert_b200"))
        shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        subprocess.check_call(["make", "-C", os.path.join(tmp, "lt_mapper_b200", "csrc"), "-j4", "-s", f"NVCC={nvcc} -DLTR_PROBE_NOMAYBE",
                               "../libltr_b200.so", "../libltr_removert.so"])
        env = dict(os.environ, LTR_PROBE_CHILD="1", PYTHONPATH=tmp)
        child = subprocess.run([sys.executable, os.path.abspath(__file__), str(kf)], env=env, capture_output=True, text=True)
        if child.returncode != 0:
            raise SystemExit(child.stderr[-4000:])
        diag = json.loads(child.stdout.strip().splitlines()[-1])
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    print("| session | alpha | map points | culled | exact [2] | full exact [5] | non-culled no-maybe share | kernel us/launch | pass ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for a, b in zip(normal, diag):
        nomaybe = b["counter1"] * 128.0 / a["pairs"]
        print(f"| {a['session']} | {a['alpha']:.3f} | {a['map_points']} | {a['culled']:.4f} | {a['exact']:.4f} | {a['exact_full']:.5f} | {nomaybe:.4f} "
              f"| {a['kernel_us_per_launch']:.0f} | {a['pass_ms']:.1f} |")
    print(json.dumps({"normal": normal, "nomaybe_build": diag}))


if __name__ == "__main__":
    main()
