"""CPU tests (no GPU, no process group) of the multi-GPU keyframe decomposition: each rank owns a contiguous keyframe block, clouds
merged over all keyframes are the rank-ordered concatenation of the per-block merges, and a pass's dynamic flags are the OR of the
per-block flags.  The arithmetic engine here is the oracle; what is under test is the decomposition the NCCL transport relies on."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_keyframe_blocks_merge_and_flag_union_equal_the_full_pass():
    """Two ranks of two keyframes each: (1) the rank-ordered concatenation of the per-block merged clouds equals the keyframe-order merge of
    all keyframes (what ltr_nccl_allgather_clouds assembles); (2) the OR of the per-block flags of an HD pass equals the single-process
    pass's flags, and neither block alone reaches it (what ltr_nccl_allreduce_flags computes)."""
    sys.path.insert(0, ROOT)
    import oracle
    import synth
    K, world = 4, 2
    blk = K // world
    full = synth.make_session(0, K, beams=12, az_steps=300)
    blocks = [synth.make_session(0, blk, beams=12, az_steps=300, k0=r * blk) for r in range(world)]   # each rank's contiguous block
    for r, mine in enumerate(blocks):
        assert np.array_equal(mine.xyzi, full.subset(r * blk, (r + 1) * blk).xyzi)
    # (1) rank-ordered concatenation of the merged clouds == keyframe-order merge
    local = [np.concatenate([oracle.transform(mine.scan(k), mine.poses[k]) for k in range(blk)]) for mine in blocks]
    expect = np.concatenate([oracle.transform(full.scan(k), full.poses[k]) for k in range(K)])
    assert np.array_equal(np.concatenate(local), expect)
    # (2) per-pass flag union: OR of the per-block flags == flags of the single-process pass
    m = oracle.voxel(expect, 0.05)
    inv = oracle.inverse_poses(full.poses)
    f_full = oracle.remove_pass(m, full.xyzi, full.offsets, inv, oracle.MODE_HD, 2.5, threads=1)
    union = np.zeros_like(f_full)
    for r, mine in enumerate(blocks):
        f_local = oracle.remove_pass(m, mine.xyzi, mine.offsets, inv[r * blk:(r + 1) * blk], oracle.MODE_HD, 2.5, threads=1)
        assert f_local.sum() < f_full.sum()   # the union really needs both blocks
        union = np.maximum(union, f_local)
    assert np.array_equal(union, f_full)


@pytest.mark.parametrize("world,split", [(1, False), (2, True), (2, False), (4, True), (8, True), (3, False), (8, False)])
def test_owned_blocks_partition_the_sessions_in_rank_order(world, split):
    """bench.owned_blocks: per session the blocks of the owning ranks are contiguous, disjoint, in rank order and cover [0, K) --
    rank-order concatenation must equal keyframe order (utility.cpp:177-189 concatenates in keyframe order)."""
    sys.path.insert(0, ROOT)
    import bench
    for K in (1000, 7, 2000):
        for s in (0, 1):
            nxt = 0
            owners = 0
            for r in range(world):
                k0, n = bench.owned_blocks(r, world, K, split)[s]
                if n == 0:
                    continue
                owners += 1
                assert k0 == nxt
                nxt = k0 + n
            assert nxt == K
            assert owners == (world // 2 if split else min(world, K))
        if split:   # a rank owns keyframes of exactly one session: ranks < world/2 the central one
            for r in range(world):
                b = bench.owned_blocks(r, world, K, split)
                assert (b[0][1] > 0) == (r < world // 2) and (b[1][1] > 0) == (r >= world // 2)
