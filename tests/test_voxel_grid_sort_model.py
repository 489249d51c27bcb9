"""The entry order of the device VoxelGrid (voxel_grid.cu) on the CPU.

voxel_grid_span (host/io.cpp) sorts its (voxel index, point index) entries with std::sort, which is not stable: the order of equal
indices decides the f32 summation order of each centroid.  The device reproduces libstdc++'s introsort instead of sorting stably.
Here:
  - `std_sort` is a transcription of libstdc++'s std::sort (__introsort_loop with _S_threshold = 16 and depth limit 2 * __lg(n),
    __move_median_to_first, __unguarded_partition, __partial_sort = make_heap + sort_heap, __final_insertion_sort).  Centroids
    summed in its order must equal the host library's bits on crafted inputs: if the toolchain's std::sort ever differs, this fails.
  - `device_sort` is the device formulation: long segments partitioned from prefix counts (the t-th position >= pivot from the left
    swaps with the t-th position <= pivot from the right while the first lies left of the second), short segments finished by the
    sequential loop, every leaf of <= 16 entries stably insertion-sorted on its own.  It must give the same permutation as `std_sort`
    on random, patterned and adversarial arrays, including ones that reach the heap-sort branch.
"""
import numpy as np
import pytest

from lt_mapper_b200 import removert

F32 = np.float32
THRESHOLD = 16
DEVICE_SMALL = 1024      # kVgSmall of voxel_grid.cu


def lg(n):
    return n.bit_length() - 1


# ------------------------------------------------------------------------------------------------------------ libstdc++ transcription
def _median_to_first(a, r, x, y, z, less):
    if less(a[x], a[y]):
        s = y if less(a[y], a[z]) else (z if less(a[x], a[z]) else x)
    elif less(a[x], a[z]):
        s = x
    elif less(a[y], a[z]):
        s = z
    else:
        s = y
    a[r], a[s] = a[s], a[r]


def _unguarded_partition(a, f, l, p, less):
    while True:
        while less(a[f], a[p]):
            f += 1
        l -= 1
        while less(a[p], a[l]):
            l -= 1
        if not f < l:
            return f
        a[f], a[l] = a[l], a[f]
        f += 1


def _adjust_heap(a, first, hole, n, value, less):
    top = hole
    c = hole
    while c < (n - 1) // 2:
        c = 2 * (c + 1)
        if less(a[first + c], a[first + c - 1]):
            c -= 1
        a[first + hole] = a[first + c]
        hole = c
    if n % 2 == 0 and c == (n - 2) // 2:
        c = 2 * (c + 1)
        a[first + hole] = a[first + c - 1]
        hole = c - 1
    parent = (hole - 1) // 2
    while hole > top and less(a[first + parent], value):
        a[first + hole] = a[first + parent]
        hole = parent
        parent = (hole - 1) // 2
    a[first + hole] = value


def _heap_sort(a, f, l, less):
    n = l - f
    if n >= 2:
        parent = (n - 2) // 2
        while True:
            _adjust_heap(a, f, parent, n, a[f + parent], less)
            if parent == 0:
                break
            parent -= 1
    while n > 1:
        n -= 1
        v = a[f + n]
        a[f + n] = a[f]
        _adjust_heap(a, f, 0, n, v, less)


def _introsort_loop(a, f, l, depth, less, trace):
    while l - f > THRESHOLD:
        if depth == 0:
            trace["heap_sorts"] += 1
            _heap_sort(a, f, l, less)
            return
        depth -= 1
        _median_to_first(a, f, f + 1, f + (l - f) // 2, l - 1, less)
        cut = _unguarded_partition(a, f + 1, l, f, less)
        _introsort_loop(a, cut, l, depth, less, trace)
        l = cut


def _final_insertion_sort(a, f, l, less):
    def insertion(f, l):
        for i in range(f + 1, l):
            v = a[i]
            if less(v, a[f]):
                a[f + 1:i + 1] = a[f:i]
                a[f] = v
            else:
                unguarded(i)

    def unguarded(i):
        v = a[i]
        while less(v, a[i - 1]):
            a[i] = a[i - 1]
            i -= 1
        a[i] = v

    if l - f > THRESHOLD:
        insertion(f, f + THRESHOLD)
        for i in range(f + THRESHOLD, l):
            unguarded(i)
    else:
        insertion(f, l)


def std_sort(items, less, trace=None):
    a = list(items)
    trace = trace if trace is not None else {"heap_sorts": 0}
    if a:
        _introsort_loop(a, 0, len(a), 2 * lg(len(a)), less, trace)
        _final_insertion_sort(a, 0, len(a), less)
    return a


def key_less(x, y):
    return x[0] < y[0]


def introsort_trace(keys):
    trace = {"heap_sorts": 0}
    std_sort([(int(k), i) for i, k in enumerate(keys)], key_less, trace)
    return trace


# ------------------------------------------------------------------------------------------------------------ device formulation
def _stable_leaf(a, f, l):
    a[f:l] = sorted(a[f:l], key=lambda e: e[0])          # Python's sort is stable


def _seq_loop(a, f, l, depth):
    """vg_introsort_seq: the loop of one thread, leaves stably sorted where they are produced."""
    stack = []
    while True:
        heaped = False
        while l - f > THRESHOLD:
            if depth == 0:
                _heap_sort(a, f, l, key_less)
                heaped = True
                break
            depth -= 1
            _median_to_first(a, f, f + 1, f + (l - f) // 2, l - 1, key_less)
            cut = _unguarded_partition(a, f + 1, l, f, key_less)
            stack.append((cut, l, depth))
            l = cut
        if not heaped:
            _stable_leaf(a, f, l)
        if not stack:
            return
        f, l, depth = stack.pop()


def _prefix_partition(a, f, l):
    """__unguarded_partition(first + 1, last, first) from prefix counts; returns the cut."""
    p = a[f][0]
    keys = np.array([e[0] for e in a[f + 1:l]], np.int64)
    pos = np.arange(f + 1, l)
    L = pos[keys >= p]                     # ascending
    R = pos[keys <= p][::-1]               # descending
    t = np.arange(min(len(L), len(R)))
    m = int(np.count_nonzero(L[t] < R[t]))
    for s in range(m):
        i, j = int(L[s]), int(R[s])
        a[i], a[j] = a[j], a[i]
    cut = int(L[m]) if m < len(L) else l
    if m > 0:
        cut = min(cut, int(R[m - 1]))
    return cut


def device_sort(keys, small=DEVICE_SMALL):
    a = [(int(k), i) for i, k in enumerate(keys)]
    n = len(a)
    big, short = [], []
    if n > small:
        big.append((0, n, 2 * lg(n)))
    elif n > 1:
        short.append((0, n, 2 * lg(n)))
    while big:
        f, l, d = big.pop()
        if d == 0:
            _heap_sort(a, f, l, key_less)
            continue
        _median_to_first(a, f, f + 1, f + (l - f) // 2, l - 1, key_less)
        cut = _prefix_partition(a, f, l)
        for cf, cl in ((cut, l), (f, cut)):
            if cl - cf > small:
                big.append((cf, cl, d - 1))
            elif cl - cf > 1:
                short.append((cf, cl, d - 1))
    for f, l, d in short:
        _seq_loop(a, f, l, d)
    return a


# ------------------------------------------------------------------------------------------------------------ adversary
def mcilroy_adversary(n):
    """M. D. McIlroy, "A killer adversary for quicksort" (1999), run against std_sort: returns keys on which it degenerates."""
    gas = n
    val = [gas] * n
    state = {"solid": 0, "candidate": 0}

    def less(x, y):
        if val[x] == gas and val[y] == gas:
            z = x if x == state["candidate"] else y
            val[z] = state["solid"]
            state["solid"] += 1
        if val[x] == gas:
            state["candidate"] = x
        elif val[y] == gas:
            state["candidate"] = y
        return val[x] < val[y]

    std_sort(list(range(n)), less)
    return np.array(val, np.int64)


def patterned(name, n, rng):
    u = np.arange(n) // 3
    return {"random": rng.integers(0, max(n // 4, 1), n), "sorted": u, "reversed": u[::-1],
            "organ_pipe": np.concatenate([u[: n // 2], u[: n - n // 2][::-1]]), "equal": np.zeros(n, np.int64),
            "few": rng.integers(0, 3, n)}[name]


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name", ["random", "sorted", "reversed", "organ_pipe", "equal", "few"])
@pytest.mark.parametrize("n", [0, 1, 2, 16, 17, 33, 100, 1500])
@pytest.mark.parametrize("small", [32, 64, DEVICE_SMALL])
def test_device_formulation_equals_transcription(name, n, small):
    rng = np.random.default_rng(n * 7 + small)
    keys = patterned(name, n, rng)
    assert device_sort(keys, small) == std_sort([(int(k), i) for i, k in enumerate(keys)], key_less)


@pytest.mark.parametrize("n", [100, 600, 3000])
@pytest.mark.parametrize("small", [32, DEVICE_SMALL])
def test_device_formulation_on_adversary(n, small):
    keys = mcilroy_adversary(n)
    assert introsort_trace(keys)["heap_sorts"] > 0, "the adversary must reach the heap-sort branch"
    assert device_sort(keys, small) == std_sort([(int(k), i) for i, k in enumerate(keys)], key_less)


def centroids_in_order(x, keys, order):
    out = []
    i = 0
    while i < len(order):
        j = i
        s = np.zeros(4, F32)
        while j < len(order) and keys[order[j]] == keys[order[i]]:
            s = (s + x[order[j]]).astype(F32)
            j += 1
        out.append(s / F32(j - i))
        i = j
    return np.array(out, F32).reshape(-1, 4)


def crafted(keys, seed):
    """One point per key on the x axis (leaf 1.0: voxel index == key); intensities 1e7 and ~1 mixed, so sums depend on the order."""
    rng = np.random.default_rng(seed)
    n = len(keys)
    x = np.zeros((n, 4), F32)
    x[:, 0] = np.asarray(keys, F32) + F32(0.5)
    x[:, 1] = rng.random(n).astype(F32) * F32(0.5)
    x[:, 2] = rng.random(n).astype(F32) * F32(0.5)
    x[:, 3] = np.where(rng.random(n) < 0.5, rng.choice([F32(1.0e7), F32(-1.0e7)], n),
                       rng.random(n).astype(F32) * F32(3.0) + F32(0.1)).astype(F32)
    return x


@pytest.mark.parametrize("case", ["random", "organ_pipe", "equal", "adversary"])
def test_transcription_matches_host_library(case):
    n = 3000
    rng = np.random.default_rng(3)
    keys = mcilroy_adversary(n) // 3 if case == "adversary" else patterned(case, n, rng)   # // 3: voxels of 3 points
    if case == "adversary":
        assert introsort_trace(keys)["heap_sorts"] > 0
    x = crafted(keys, 9)
    host, ov = removert.voxel_grid(x, 1.0)
    assert not ov
    order = [e[1] for e in std_sort([(int(k), i) for i, k in enumerate(keys)], key_less)]
    mine = centroids_in_order(x, keys, order)
    assert mine.shape == host.shape and np.array_equal(mine.view(np.uint32), host.view(np.uint32)), \
        "the toolchain's std::sort no longer matches the libstdc++ transcription"
    stable = centroids_in_order(x, keys, list(np.argsort(keys, kind="stable")))
    assert not np.array_equal(stable.view(np.uint32), host.view(np.uint32)), "input does not tell the permutations apart"
