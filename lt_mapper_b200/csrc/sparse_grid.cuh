// Sparse (segment, cell) grid levels of the exact nearest-neighbour searches (scanside.cu builds them; icp.cu searches them too).
// A level sorts its points by the 64-bit key (segment, cz, cy, cx) with the project's radix sort (util.cu) and keeps the sorted unique
// keys, each cell's first point and the points in key order, with the point's index in the input as the bits of float4::w.  The sort
// is stable and starts from ascending input indices, so the points of one cell are in ascending index order.  A row of cells (one
// segment, cz, cy; consecutive cx) is one contiguous key range: one binary search per row.
//
// Shell search (shell_search below).  A query searches shell by shell (Chebyshev radius s = 0, 1, ... in cells around its own cell) and
// stops after shell s when the block holds every cell of the level, or when its accumulator settles.  Both accumulators settle on the
// bound B(s) = ((s - 2^-6) c)^2 (1 - 2^-20) (c = 1 / inv_cell, the cell side the indices are computed with), for s >= 1.
// Why B(s) is exact.  A point p outside the block lies in a cell whose index differs from the query's by >= s + 1 on some axis a.
// Both indices are floor(fl(fl(v - origin) * inv_cell)) with |.| clamped to 2^40 (a clamp only moves a query's index towards the box, so
// its true distance is larger still); each evaluation carries a relative error below 3 * 2^-53, i.e. below 2^-11 cells for |index| <= 2^40,
// so |p_a - q_a| >= (s - 2^-10) c > (s - 2^-6) c in exact arithmetic.  FLANN's L2_Simple in f32 (((dx*dx) + dy*dy) + dz*dz, no FMA):
// rounding is monotone, so |dx| = |fl(q_a - p_a)| >= fl((s - 2^-6) c) >= (s - 2^-6) c (1 - u), u = 2^-24, fl(dx*dx) >= dx^2 (1 - u), and the
// two additions of non-negative terms round to no less than fl(dx*dx).  The computed distance of every point outside the block is
// therefore >= ((s - 2^-6) c)^2 (1 - u)^3 > B(s): STRICTLY greater than B(s).
//  * k smallest values (scanside.cu, Best<K> over ref_math.cuh's TopK): once the k-th smallest computed distance D_k <= B(s), no point outside the block can
//    displace a value of the k smallest (a tie at D_k leaves the multiset unchanged), so the double sum in ascending order, its float
//    rounding and the division by float(k) are final.  D_k = 0 cannot be undercut by any distance, so it settles in any shell, shell 0
//    included.  How many values enter the sum is min(k, points evaluated), never "finite ones": an overflowed +inf distance is summed as
//    FLANN would return it.
//  * nearest point with the lowest index on ties (icp.cu, Nearest): once the smallest distance D <= B(s), every point at distance D is
//    inside the block and has been evaluated, so the lowest index among them is the lowest overall.  D = 0 does not settle early: an
//    underflowed 0 can sit in the next cell, and its index may be lower.
// Bounded levels give up after max_shell shells and the query moves to the next, 4x coarser level; the coarsest level (at most
// kGridFinalDim cells per axis) searches until the rule holds.  Which level answers changes the cost only.
#pragma once
#include "ltr_internal.cuh"
#include "ref_math.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace ltr {

constexpr int kGridCellBits = 17;                         // per axis: indices < 2^17
constexpr int kGridSegShift = 3 * kGridCellBits;          // 51: segment above the three cell indices
constexpr int kGridMaxSegments = 1 << (64 - kGridSegShift);   // 8192 segments per level
constexpr int kGridMaxDim = (1 << kGridCellBits) - 1;
constexpr double kGridCell0 = 0.25;                       // finest cell side [m]
constexpr double kGridLevelRatio = 4.0;
constexpr int kGridMaxLevels = 8;
constexpr int kGridFinalDim = 10;                         // a level of at most this many cells per axis is searched without a shell bound

struct Level {
    double origin[3];
    double inv_cell, cell;          // cell = 1 / inv_cell
    int dim[3];
    int final_level;
    const unsigned long long* keys; // sorted unique (segment, cell) keys
    const uint32_t* start;          // first point of each cell, [ncell] = number of points
    const float4* pts;              // points in key order, w = __uint_as_float(input index)
    const uint32_t* seg_first;      // cells of segment s: [seg_first[s], seg_first[s + 1])
};

struct LevelBuf {
    Level L{};
    void* block = nullptr;
};

__device__ __forceinline__ unsigned long long cell_key(int seg, long long cx, long long cy, long long cz) {
    return ((unsigned long long)seg << kGridSegShift) | ((unsigned long long)cz << (2 * kGridCellBits)) |
           ((unsigned long long)cy << kGridCellBits) | (unsigned long long)cx;
}

__device__ __forceinline__ long long cell_index(double v, double origin, double inv_cell) {
    const double t = fmin(fmax((v - origin) * inv_cell, -0x1p40), 0x1p40);
    return (long long)floor(t);
}

// B(s) of the header: every point outside the block of shell s has a computed distance strictly greater than this
__device__ __forceinline__ double shell_bound(long long s, double cell) {
    const double r = ((double)s - 0x1p-6) * cell;
    return r * r * (1.0 - 0x1p-20);
}

// the points L.pts[*s, *e) of the cells [xa, xb] of row (y, z) of segment seg (cells [c0, c1) of the level), in key order
__device__ __forceinline__ void row_points(const Level& L, uint32_t c0, uint32_t c1, int seg, long long xa, long long xb, long long y, long long z,
                                           uint32_t* s, uint32_t* e) {
    const unsigned long long ka = cell_key(seg, xa, y, z), kb = cell_key(seg, xb, y, z);
    uint32_t lo = c0, hi = c1;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (L.keys[mid] < ka) lo = mid + 1; else hi = mid; }
    uint32_t ci = lo;
    while (ci < c1 && L.keys[ci] <= kb) ++ci;
    *s = L.start[lo];
    *e = L.start[ci];
}

// the cells [xa, xb] of row (y, z) of segment seg (cells [c0, c1) of the level): acc.push(distance, point) in key order
template <class Acc>
__device__ __forceinline__ void shell_row(const Level& L, uint32_t c0, uint32_t c1, int seg, long long xa, long long xb, long long y, long long z,
                                          float qx, float qy, float qz, Acc& acc) {
    const unsigned long long ka = cell_key(seg, xa, y, z), kb = cell_key(seg, xb, y, z);
    uint32_t lo = c0, hi = c1;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (L.keys[mid] < ka) lo = mid + 1; else hi = mid; }
    for (uint32_t ci = lo; ci < c1 && L.keys[ci] <= kb; ++ci) {
        const uint32_t e = L.start[ci + 1];
        for (uint32_t p = L.start[ci]; p < e; ++p) {
            const float4 t = L.pts[p];
            acc.push(l2_simple(qx, qy, qz, t.x, t.y, t.z), t);
        }
    }
}

// The shell search of the header over the points of segment seg: Acc has push(float d, float4 point) and settled(long long s, double cell),
// the stop rule after shell s.  false: not settled within max_shell shells on a bounded level.
template <class Acc>
__device__ __forceinline__ bool shell_search(const Level& L, int seg, float qx, float qy, float qz, int max_shell, Acc& acc) {
    const float q[3] = {qx, qy, qz};
    long long c[3], s0 = 0, cover = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        c[d] = cell_index((double)q[d], L.origin[d], L.inv_cell);
        const long long hi = (long long)L.dim[d] - 1;
        s0 = max(s0, max(-c[d], c[d] - hi));       // Chebyshev distance from the query's cell to the box: nearer shells are empty
        cover = max(cover, max(c[d], hi - c[d]));  // from this radius on the block holds every cell
    }
    const uint32_t c0 = L.seg_first[seg], c1 = L.seg_first[seg + 1];
    bool done = c0 == c1;
    for (long long s = s0; !done; ++s) {
        if (!L.final_level && s > max_shell) return false;
        const long long z0 = max(c[2] - s, 0ll), z1 = min(c[2] + s, (long long)L.dim[2] - 1);
        const long long y0 = max(c[1] - s, 0ll), y1 = min(c[1] + s, (long long)L.dim[1] - 1);
        const long long xa = max(c[0] - s, 0ll), xb = min(c[0] + s, (long long)L.dim[0] - 1);
        for (long long z = z0; z <= z1; ++z) {
            const bool zface = z == c[2] - s || z == c[2] + s;
            for (long long y = y0; y <= y1; ++y) {
                if (zface || y == c[1] - s || y == c[1] + s) {
                    if (xa <= xb) shell_row(L, c0, c1, seg, xa, xb, y, z, qx, qy, qz, acc);
                } else {
                    if (c[0] - s >= 0 && c[0] - s < L.dim[0]) shell_row(L, c0, c1, seg, c[0] - s, c[0] - s, y, z, qx, qy, qz, acc);
                    if (s > 0 && c[0] + s >= 0 && c[0] + s < L.dim[0]) shell_row(L, c0, c1, seg, c[0] + s, c[0] + s, y, z, qx, qy, qz, acc);
                }
            }
        }
        if (s >= cover) break;
        done = acc.settled(s, L.cell);
    }
    return true;
}

// Grid level of cell side `cell` over the points of p (segments from d_off, or one segment when d_off is null), box [mn, mx] of p
// (scanside.cu).  *out owns one allocation of the context's allocator.
int build_level(ltr_ctx* ctx, PtrView p, const int64_t* d_off, int nseg, const float mn[3], const float mx[3], double cell, bool final_level,
                LevelBuf* out);

// The levels of one point set, finest first (cell sides cell0 * 4^l), built as far as some query needs them; freed by release() or the
// destructor.
struct Pyramid {
    ltr_ctx* ctx;
    PtrView pts{nullptr, nullptr, nullptr, nullptr, 0};
    const int64_t* d_off = nullptr;
    int nseg = 1;
    float mn[3], mx[3];
    double cell0 = kGridCell0;
    std::vector<LevelBuf> levels;

    explicit Pyramid(ltr_ctx* c) : ctx(c) {}
    ~Pyramid() { release(); }
    Pyramid(const Pyramid&) = delete;
    Pyramid& operator=(const Pyramid&) = delete;
    void init(PtrView p, const int64_t* off, int ns, const float lo[3], const float hi[3]) {
        pts = p; d_off = off; nseg = ns;
        double ext = 0.0;
        for (int d = 0; d < 3; ++d) { mn[d] = lo[d]; mx[d] = hi[d]; ext = std::max(ext, (double)hi[d] - (double)lo[d]); }
        cell0 = std::max(kGridCell0, ext / (double)(kGridMaxDim - 4));   // indices < 2^17 on the finest level
    }
    int get(int l, const Level** out) {
        while ((int)levels.size() <= l) {
            const int m = (int)levels.size();
            const double cell = cell0 * std::pow(kGridLevelRatio, m);
            int dmax = 0;
            for (int d = 0; d < 3; ++d) dmax = std::max(dmax, (int)std::floor(((double)mx[d] - (double)mn[d]) / cell) + 3);
            LevelBuf b;
            LTR_TRY(build_level(ctx, pts, d_off, nseg, mn, mx, cell, dmax <= kGridFinalDim || m == kGridMaxLevels - 1, &b));
            levels.push_back(b);
        }
        *out = &levels[(size_t)l].L;
        return LTR_OK;
    }
    void release() { for (auto& b : levels) if (b.block) dev_free(ctx, b.block); levels.clear(); }
};

}  // namespace ltr
