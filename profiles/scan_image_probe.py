"""Scan-side image work of the remove / revert / ND / PD passes in one steady-state configs[2] step: `python profiles/scan_image_probe.py [KF]`.

Runs Step 0 and one warm-up step (Step 1 + static projection + Step 2), then profiles one more step with `torch.profiler` (CUDA
activities) and splits its kernel list into the 24 `ltr_remove_pass` calls: once the current pass has launched its projection, the next
begins at a scan-image build (a `fill_u32_kernel` followed by `scan_rimg*_kernel`) or at a winner-image fill (`fill_u64_kernel`)
followed by an image kernel, whichever comes first.  For each pass it prints the device time of the
scan-side image kernels (fills of the scan / approximate-minimum images, `scan_rimg*_kernel`, `scan_window_max_kernel`,
`scan_test_image_kernel`) next to the projection and resolve kernels, then the totals per step.  The pass names come from the
step's pass log.  Profiling slows the host, not the kernels; the step time it prints is not a bench value."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lt_mapper_b200 import removert  # noqa: E402

IMAGE = ("fill_u32_kernel", "scan_rimg_kernel", "scan_rimg_fast_kernel", "scan_window_max_kernel", "scan_test_image_kernel")
PROJECT = ("map_project_fast_kernel", "map_project_kernel", "deferred_resolve_kernel", "resolve_kernel", "tile_sphere_kernel")


def short(name):
    n = name.split("(")[0].replace("void ", "")
    n = n.split("<")[0]
    return n.split("::")[-1]


def main():
    kf = int(sys.argv[1]) if len(sys.argv) > 1 else bench.KF_PER_SESSION
    p = torch.cuda.get_device_properties(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# {p.name}; nvidia-smi: {q}")
    blocks = bench.gen_block(0, kf)
    R = removert.Removerter(num_knn=bench.NUM_KNN, knn_thr=bench.KNN_THR, schedule=bench.schedule())
    for s, (d, inv) in enumerate(blocks):
        R.load_session(s, d.xyzi, d.offsets, d.poses, inv)
    R.run_step0()
    R.run_step12()
    R.reset_to_step0()
    R.ctx.synchronize()
    l0 = R.ctx.kernel_launches()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        R.run_step12()
        R.ctx.synchronize()
    launches = R.ctx.kernel_launches() - l0
    log = R.log()
    R.close()
    kernels = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.name and "emset" not in e.name),
                     key=lambda e: e.time_range.start)
    names = [short(e.name) for e in kernels]
    passes = []   # per pass: {kernel: [us, launches]}
    cur = None
    for i, (e, n) in enumerate(zip(kernels, names)):
        nxt = names[i + 1] if i + 1 < len(names) else ""
        starts = (n == "fill_u64_kernel" and nxt in IMAGE) or (n == "fill_u32_kernel" and nxt.startswith("scan_rimg"))
        if starts and (cur is None or "map_project_fast_kernel" in cur or "map_project_kernel" in cur):
            cur = {}
            passes.append(cur)
        if cur is not None and (n in IMAGE or n in PROJECT):
            a = cur.setdefault(n, [0.0, 0])
            a[0] += e.time_range.elapsed_us()
            a[1] += 1
    total_us = sum(e.time_range.elapsed_us() for e in kernels)
    pass_names = [r.get("what", r.get("name", "?")) if isinstance(r, dict) else str(r[0]) for r in log]
    print(f"{len(passes)} remove passes found, {len(pass_names)} in the pass log; kernel time in the step {total_us / 1e3:.1f} ms, "
          f"{len(kernels)} kernels ({launches} counted by the library)")
    cols = IMAGE + ("map_project_fast_kernel", "resolve_kernel", "deferred_resolve_kernel")
    print("| pass | " + " | ".join(cols) + " | image total |")
    print("|---|" + "---|" * (len(cols) + 1))
    tot = {}
    per_kind = {}
    for i, ps in enumerate(passes):
        name = pass_names[i] if i < len(pass_names) else "?"
        img = sum(ps.get(k, [0, 0])[0] for k in IMAGE)
        per_kind[name] = per_kind.get(name, 0.0) + img
        for k, v in ps.items():
            t = tot.setdefault(k, [0.0, 0])
            t[0] += v[0]; t[1] += v[1]
        print(f"| {i} {name} | " + " | ".join(f"{ps.get(k, [0, 0])[0]:.0f} ({ps.get(k, [0, 0])[1]})" for k in cols) + f" | {img:.0f} |")
    img_total = sum(tot.get(k, [0, 0])[0] for k in IMAGE)
    print(f"image-side kernels per step: {img_total / 1e3:.1f} ms; per pass kind (ms): " + ", ".join(f"{k} {v / 1e3:.1f}" for k, v in per_kind.items()))
    print(json.dumps({"gpu": p.name, "nvidia_smi": q, "passes": len(passes), "kernel_ms": round(total_us / 1e3, 2), "kernels": len(kernels),
                      "library_launches": launches, "image_ms": round(img_total / 1e3, 2),
                      "per_kernel_us": {k: [round(v[0], 1), v[1]] for k, v in sorted(tot.items())},
                      "image_ms_per_pass_kind": {k: round(v / 1e3, 2) for k, v in per_kind.items()}}))


if __name__ == "__main__":
    main()
