"""The host orchestrator's error paths: a stage or a delta-map call that fails half-way (a non-finite coordinate reaching the voxeliser
or the per-keyframe kNN split) releases every handle it created, so repeating it in a long-lived Removerter leaves the context's live
bytes where they were."""
import numpy as np
import pytest

import synth
import lt_mapper_b200 as ltr
from lt_mapper_b200 import removert

pytestmark = pytest.mark.gpu
UNSUPPORTED = -3


@pytest.fixture(scope="module")
def pair():
    return synth.make_pair(4, beams=16, az_steps=600)


def _load(R, sess, d, nan_kf=None):
    xyzi = d.xyzi.copy()
    if nan_kf is not None:
        xyzi[d.offsets[nan_kf] + 7, 0] = np.nan
    R.load_session(sess, xyzi, d.offsets, d.poses, removert.inverse_poses(d.poses))


def _live_handles(ctx, n=256):
    """(clouds, scan sets) the context holds.  A reload may take cached blocks up to a quarter larger than it asks for, so live bytes
    differ between attempts that hold the same handles; a leak shows as a handle that stays live."""
    def live(probe):
        try:
            probe()
            return 1
        except ltr.LtrError:
            return 0
    return (sum(live(lambda: ctx.cloud_size(h)) for h in range(n)), sum(live(lambda: ctx.scanset_info(h)) for h in range(n)))


@pytest.mark.parametrize("nan_sess", [0, 1])
def test_step0_with_a_non_finite_coordinate_leaks_nothing(pair, nan_sess):
    """makeGlobalMap: the voxeliser rejects the merged cloud of the session with the NaN, after the merged cloud exists."""
    with removert.Removerter() as R:
        live = []
        for _ in range(3):
            for sess, d in enumerate(pair):
                _load(R, sess, d, nan_kf=2 if sess == nan_sess else None)
            with pytest.raises(ltr.LtrError) as e:
                R.run_step0()
            assert e.value.code == UNSUPPORTED
            live.append(_live_handles(R.ctx))
        assert live == [live[0]] * 3


def _generation(rng, K, bad):
    """One generation's (PD, ND) per keyframe; bad: a non-finite point in PD's keyframe 1."""
    sets = []
    for _ in range(2):
        sizes = rng.integers(30, 80, K)
        pts = np.concatenate([rng.uniform(-20, 20, (int(sizes.sum()), 3)), rng.random((int(sizes.sum()), 1))], 1).astype(np.float32)
        sets.append((pts, np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)))
    if bad:
        pts, off = sets[0]
        pts[off[1] + 3, 2] = np.inf
    return sets


@pytest.mark.parametrize("bad_gen", [1, 2])
def test_delta_maps_with_a_non_finite_point_leak_nothing(pair, bad_gen):
    """compose_changes / rollback over three generations fail in the fold of generation bad_gen (generation 2: after generation 1 was
    already composed) and release what they built."""
    c, _ = pair
    rng = np.random.default_rng(bad_gen)
    with removert.Removerter() as R:
        _load(R, 0, c)
        R.set_delta_maps(True)
        for g in range(3):
            (pd, pd_off), (nd, nd_off) = _generation(rng, c.K, g == bad_gen)
            R.delta_load(pd, pd_off, nd, nd_off)
        for call in (lambda: R.compose_changes(0, 3), lambda: R.rollback(0)):
            before = R.ctx.memory_stats()[0]
            with pytest.raises(ltr.LtrError) as e:
                call()
            assert e.value.code == UNSUPPORTED
            assert R.ctx.memory_stats()[0] == before
