// Sparse (segment, cell) grid levels of the exact nearest-neighbour searches (scanside.cu builds them; icp.cu searches them too).
// A level sorts its points by the 64-bit key (segment, cz, cy, cx) with the project's radix sort (util.cu) and keeps the sorted unique
// keys, each cell's first point and the points in key order, with the point's index in the input as the bits of float4::w.  The sort
// is stable and starts from ascending input indices, so the points of one cell are in ascending index order.  The exactness proof of
// the shell search over these levels is in scanside.cu's header.
#pragma once
#include "ltr_internal.cuh"
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

// Grid level of cell side `cell` over the points of p (segments from d_off, or one segment when d_off is null), box [mn, mx] of p
// (scanside.cu).  *out owns one allocation of the context's allocator.
int build_level(ltr_ctx* ctx, PtrView p, const int64_t* d_off, int nseg, const float mn[3], const float mx[3], double cell, bool final_level,
                LevelBuf* out);

// The levels of one point set, finest first (cell sides cell0 * 4^l), built as far as some query needs them.
struct Pyramid {
    PtrView pts{nullptr, nullptr, nullptr, nullptr, 0};
    const int64_t* d_off = nullptr;
    int nseg = 1;
    float mn[3], mx[3];
    double cell0 = kGridCell0;
    std::vector<LevelBuf> levels;

    void init(PtrView p, const int64_t* off, int ns, const float lo[3], const float hi[3]) {
        pts = p; d_off = off; nseg = ns;
        double ext = 0.0;
        for (int d = 0; d < 3; ++d) { mn[d] = lo[d]; mx[d] = hi[d]; ext = std::max(ext, (double)hi[d] - (double)lo[d]); }
        cell0 = std::max(kGridCell0, ext / (double)(kGridMaxDim - 4));   // indices < 2^17 on the finest level
    }
    int get(ltr_ctx* ctx, int l, const Level** out) {
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
    void release(ltr_ctx* ctx) { for (auto& b : levels) if (b.block) dev_free(ctx, b.block); levels.clear(); }
};

}  // namespace ltr
