"""Worker of tests/test_gpu_delta_multi.py: one rank of a torchrun job (or a single process) runs a two-generation in-memory cascade with
delta maps on (sessions 0 -> 1 -> 2 of synth), then composes and rolls back, and writes the SHA-256 of every composed / restored
per-keyframe cloud and of the restored map it holds to <out>/rank<r>.json.  Keys carry GLOBAL keyframe indices, so the files of all
ranks of a run can be merged and compared with the single-process run."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def dg(a):
    a = np.ascontiguousarray(a)
    return [int(len(a)), hashlib.sha256(a.tobytes()).hexdigest()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--kf", type=int, default=6)
    ap.add_argument("--split", type=int, default=1)
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local = int(os.environ.get("LOCAL_RANK", "0"))
    import torch
    import bench
    import synth
    from lt_mapper_b200 import removert
    torch.cuda.set_device(local)
    split = bool(args.split) and world >= 2 and world % 2 == 0
    R = removert.Removerter(device=local, num_knn=2, knn_thr=0.01)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        ids = [removert.nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        R.init_nccl(ids[0], rank, world, split_sessions=split)
    own = bench.owned_blocks(rank, world, args.kf, split)
    empty = (np.zeros((0, 4), np.float32), np.zeros(1, np.int64), np.zeros((0, 4, 4)), np.zeros((0, 4, 4)))

    def load(slot, session):
        k0, n = own[slot]
        if n == 0:
            R.load_session(slot, *empty)
            return
        d = synth.make_session(session, n, k0=k0, beams=16, az_steps=600, threads=2)
        R.load_session(slot, d.xyzi, d.offsets, d.poses, removert.inverse_poses(d.poses))

    R.set_delta_maps(True)
    load(0, 0)
    for session in (1, 2):    # session 2 has every car: it brings back what session 1 removed
        load(1, session)
        R.run_step0(); R.run_step12(); R.run_step3()
        R.cascade_promote_updated()
    out = {"delta_count": R.delta_count()}

    def scans(tag, name):
        try:
            pts, off = R.scanset(name, 0)
        except Exception:  # noqa: BLE001 -- not held by this rank
            return
        for k in range(len(off) - 1):
            out[f"{tag}:{own[0][0] + k}"] = dg(pts[off[k]:off[k + 1]])

    for i, j in ((0, 1), (1, 2), (0, 2)):
        R.compose_changes(i, j)
        scans(f"composed_pd[{i},{j})", "composed_pd_")
        scans(f"composed_nd[{i},{j})", "composed_nd_")
    for i in (0, 1, 2):
        R.rollback(i)
        scans(f"restored{i}", "keyframe_scans_restored_")
        try:
            out[f"restored_map{i}"] = dg(R.cloud("saved:restored_map"))
        except Exception:  # noqa: BLE001 -- no central keyframes on this rank
            pass
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, f"rank{rank}.json"), "w") as f:
        json.dump(out, f)
    R.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
