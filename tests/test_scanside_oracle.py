"""The CPU restatement of scan-side removal (tests/_scanside_oracle.py) and the exact k-NN sums it is built on."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle
import _scanside_oracle as so

NANOFLANN = os.path.join(os.path.dirname(oracle.__file__), os.pardir, os.pardir, "reference", "ltslam", "include", "ltslam", "nanoflann.hpp")


def _brute_sums(q, t, k):
    """FLANN L2_Simple evaluated op by op in float32 (((dx*dx) + dy*dy) + dz*dz), k smallest, summed ascending in float64."""
    q = np.asarray(q, np.float32)[:, :3]
    t = np.asarray(t, np.float32)[:, :3]
    dx = q[:, None, 0] - t[None, :, 0]
    dy = q[:, None, 1] - t[None, :, 1]
    dz = q[:, None, 2] - t[None, :, 2]
    d = ((dx * dx) + (dy * dy)) + (dz * dz)
    assert d.dtype == np.float32
    d.sort(axis=1)
    s = np.zeros(len(q), np.float64)
    for j in range(min(k, t.shape[0])):
        s = s + d[:, j].astype(np.float64)
    return s


def _cloud(rng, n, dup):
    c = np.zeros((n, 4), np.float32)
    c[:, :3] = rng.normal(0.0, 3.0, (n, 3)).astype(np.float32)
    if dup and n > 4:
        idx = rng.integers(0, n, n // 4)
        c[rng.integers(0, n, n // 4)] = c[idx]        # exact duplicates
    c[:, 3] = rng.uniform(0, 100, n).astype(np.float32)
    return c


@pytest.mark.parametrize("k", [1, 2, 3, 5, 16])
@pytest.mark.parametrize("n_target", [1, 4, 15, 700])
def test_exact_knn_sums_equal_brute_force(k, n_target):
    rng = np.random.default_rng(1000 * k + n_target)
    t = _cloud(rng, n_target, dup=True)
    q = np.concatenate([_cloud(rng, 300, dup=False), t[: min(50, n_target)]])    # queries on target points: distance 0 first
    exp_sum = _brute_sums(q, t, k)
    got = oracle.knn_dists(q, t, k)
    s = np.zeros(len(q), np.float64)
    for j in range(min(k, n_target)):
        s = s + got[:, j].astype(np.float64)
    assert np.array_equal(s, exp_sum)
    avg = so.knn_avg(q, t, k)
    assert np.array_equal(avg.view(np.uint32), (exp_sum.astype(np.float32) / np.float32(k)).view(np.uint32))


def test_self_knn_counts_the_query_and_its_duplicates():
    c = np.array([[0, 0, 0, 0], [0, 0, 0, 1], [1, 0, 0, 0], [0, 2, 0, 0]], np.float32)
    avg = so.knn_avg(c, c, 3)
    # point 0: itself, its duplicate, then (1,0,0) -> (0 + 0 + 1) / 3
    assert avg[0] == np.float32(1.0) / np.float32(3)
    # a target smaller than k contributes all of its points and is still divided by k
    assert so.knn_avg(c[:1], c[2:3], 4)[0] == np.float32(0.25)


def test_criteria_on_a_hand_built_scan():
    """map: static iff |avg_map| < thr; scan minus map: static iff |avg_scan - avg_map| < thr (f32)."""
    m = np.array([[0, 0, 0, 0], [0.1, 0, 0, 0], [20, 0, 0, 0], [20.1, 0, 0, 0]], np.float32)
    scan = np.array([[0.05, 0, 0, 0], [20, 0.1, 0, 0], [50, 0, 0, 0], [50.1, 0, 0, 0]], np.float32)
    eye = np.eye(4)
    st, dy, mask = so.split_scan(scan, eye, eye, m, so.MAP, 1, 0.05)
    assert list(mask) == [True, True, False, False] and len(st) == 2 and len(dy) == 2
    # k = 2: the near points' own second neighbour is ~400 m^2 away (avg_scan ~ 200) while avg_map is small; the far pair has
    # avg_scan = 0.005 against avg_map ~ 900: every difference exceeds thr
    st, dy, mask = so.split_scan(scan, eye, eye, m, so.SCAN_MINUS_MAP, 2, 1.0)
    assert not mask.any() and len(dy) == 4
    # a scan that is the map itself: both averages are equal, every point is static
    st, dy, mask = so.split_scan(m, eye, eye, m, so.SCAN_MINUS_MAP, 2, 1e-6)
    assert mask.all() and np.array_equal(st, m)
    with pytest.raises(ValueError):
        so.split_scan(scan, eye, eye, m[:0], so.MAP, 1, 0.05)


def test_split_round_trips_through_the_pose():
    rng = np.random.default_rng(5)
    scan = _cloud(rng, 200, dup=True)
    a = 0.3
    pose = np.array([[np.cos(a), -np.sin(a), 0, 4.0], [np.sin(a), np.cos(a), 0, -2.0], [0, 0, 1, 0.5], [0, 0, 0, 1]])
    inv = oracle.inverse4x4(pose)
    m = so.local2global(scan, pose)[::3]
    st, dy, mask = so.split_scan(scan, pose, inv, m, so.SCAN_MINUS_MAP, 3, 0.5)
    assert len(st) + len(dy) == len(scan) and len(st) == int(mask.sum())
    assert np.allclose(st[:, :3], scan[mask, :3], atol=1e-4)
    assert np.array_equal(st[:, 3], scan[mask, 3])


@pytest.mark.skipif(not os.path.exists(NANOFLANN) or shutil.which("g++") is None, reason="the reference's vendored nanoflann is not available")
@pytest.mark.parametrize("k", [1, 2, 3, 5, 16])
def test_exact_knn_against_vendored_nanoflann(tmp_path, k):
    """The oracle's k smallest distances equal nanoflann's KDTreeSingleIndexAdaptor (L2_Simple_Adaptor<float>) on clouds with duplicates."""
    src = tmp_path / "nf.cpp"
    src.write_text(r'''
#include <cstdio>
#include <vector>
#include "nanoflann.hpp"
struct Cloud { std::vector<float> p; size_t kdtree_get_point_count() const { return p.size() / 3; }
  float kdtree_get_pt(size_t i, size_t d) const { return p[3 * i + d]; } template <class B> bool kdtree_get_bbox(B&) const { return false; } };
int main(int argc, char** argv) {
  int n, m, k; FILE* f = std::fopen(argv[1], "rb"); std::fread(&n, 4, 1, f); std::fread(&m, 4, 1, f); std::fread(&k, 4, 1, f);
  Cloud t; t.p.resize(3 * (size_t)n); std::fread(t.p.data(), 4, t.p.size(), f); std::vector<float> q(3 * (size_t)m); std::fread(q.data(), 4, q.size(), f); std::fclose(f);
  typedef nanoflann::KDTreeSingleIndexAdaptor<nanoflann::L2_Simple_Adaptor<float, Cloud>, Cloud, 3> Tree;
  Tree tree(3, t, nanoflann::KDTreeSingleIndexAdaptorParams(15)); tree.buildIndex();
  FILE* o = std::fopen(argv[2], "wb");
  for (int i = 0; i < m; ++i) { std::vector<size_t> idx(k); std::vector<float> d(k, 0.0f);
    size_t got = tree.knnSearch(&q[3 * (size_t)i], k, idx.data(), d.data()); for (size_t j = got; j < (size_t)k; ++j) d[j] = 1.0f / 0.0f;
    std::fwrite(d.data(), 4, k, o); }
  std::fclose(o); return 0; }
''')
    exe = tmp_path / "nf"
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++14", "-I", os.path.dirname(os.path.abspath(NANOFLANN)), "-o", str(exe), str(src)])
    rng = np.random.default_rng(77 + k)
    t = _cloud(rng, 3000, dup=True)
    q = np.concatenate([_cloud(rng, 500, dup=False), t[:100]])
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        np.array([len(t), len(q), k], np.int32).tofile(f)
        np.ascontiguousarray(t[:, :3]).tofile(f)
        np.ascontiguousarray(q[:, :3]).tofile(f)
    subprocess.check_call([str(exe), str(inp), str(tmp_path / "out.bin")])
    ref = np.fromfile(tmp_path / "out.bin", np.float32).reshape(len(q), k)
    assert np.array_equal(ref.view(np.uint32), oracle.knn_dists(q, t, k).view(np.uint32))
