// Tile-level occlusion / range culling for the scan-minus-map variants (HD / revert / PD) of the map projection.
//
// Map clouds come out of the voxeliser in octree (Morton) order, so 128 consecutive points form a compact patch
// (median radius 0.6 m on the BASELINE maps).  For a tile with bounding sphere (c, rho) and a keyframe with origin o:
// every point p of the tile has range >= |c - o| - rho and lies inside the cone of half-angle asin(rho / |c - o|) around
// c - o, hence inside a pixel rectangle around the pixel of c.  If
//        max over that rectangle of the scan range image  <=  (|c - o| - rho) + thres - margin
// then scan(px_p) - range_p <= thres for every p in the tile: no point of the tile is a candidate (SURVEY.md A.2), so all
// 128 (point, keyframe) pairs are skipped.  This removes the map regions that are occluded in, or beyond the reach of, a
// keyframe's scan (~30 % of all pairs on the BASELINE scene) and never changes a result.  The rectangle maximum comes
// from sliding-window maxima of the scan image (a 2-D sparse table, windows of 2..32 pixels): four overlapping windows cover a
// near-square rectangle exactly.  The 32 tests of one tile against the 32
// keyframes of a launch are evaluated by the 32 lanes of the warp in parallel (one keyframe per lane) and exchanged with
// one ballot, so the test costs ~1 % of the work it saves.
//
// Not applicable to the true-min variants (ND, visible points): there a far, otherwise invisible point still wins its pixel.
#pragma once
// included from the middle of project_fast.cuh (needs FastCfg / fast_project, is needed by map_project_fast_kernel)

namespace ltr {

constexpr int kPyrLevels = 5;  // sliding-window maxima of 2x2, 4x4, 8x8, 16x16 and 32x32 pixels

struct CullArgs {
    const float4* tiles;        // per 128-point tile: sphere centre xyz, radius (inflated)
    long long ntiles;
    const float* pyr;           // [keyframes in launch][kPyrLevels][rows * cols]: level L at pixel (r, c) = max of the scan range over the
                                // 2^L x 2^L window starting there (cut at the image edge), empty pixel -> empty_value
    unsigned pyr_stride;        // kPyrLevels * rows * cols
    int enabled;
};

constexpr int kTilePts = 128;   // points per tile == the points one warp of map_project_fast_kernel owns (32 lanes x 4)

// bounding sphere of each 128-point tile: one warp per tile, 4 points per lane
__global__ void __launch_bounds__(256) tile_sphere_kernel(PtrView map, float4* __restrict__ tiles, long long ntiles) {
    const long long tile = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (tile >= ntiles) return;
    const unsigned lane = threadIdx.x & 31;
    float px[4], py[4], pz[4];
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int64_t i = min((int64_t)tile * kTilePts + j * 32 + lane, map.n - 1);   // padding repeats the last point (inside the last tile)
        px[j] = map.x[i]; py[j] = map.y[i]; pz[j] = map.z[i];
        lo[0] = fminf(lo[0], px[j]); lo[1] = fminf(lo[1], py[j]); lo[2] = fminf(lo[2], pz[j]);
        hi[0] = fmaxf(hi[0], px[j]); hi[1] = fmaxf(hi[1], py[j]); hi[2] = fmaxf(hi[2], pz[j]);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d)
        for (int o = 16; o > 0; o >>= 1) {
            lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
            hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
        }
    const float cx = 0.5f * (lo[0] + hi[0]), cy = 0.5f * (lo[1] + hi[1]), cz = 0.5f * (lo[2] + hi[2]);
    float r2 = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float dx = px[j] - cx, dy = py[j] - cy, dz = pz[j] - cz; r2 = fmaxf(r2, dx * dx + dy * dy + dz * dz); }
    for (int o = 16; o > 0; o >>= 1) r2 = fmaxf(r2, __shfl_xor_sync(0xffffffffu, r2, o));
    if (lane == 0) tiles[tile] = make_float4(cx, cy, cz, sqrtf(r2) * 1.00001f + 1.0e-4f);   // inflated: f32 rounding of centre / distance
}

// Sliding-window maxima (a 2-D sparse table) of the scan range images of one launch: level L at (r, c) is the maximum of the scan range
// over the 2^L x 2^L window starting at (r, c), cut at the image edge (10000.0f = empty -> empty_value).  One CTA per 32 x 32 output
// pixels of one keyframe: it loads the 63 x 63 pixels those windows reach (-inf beyond the edge, which is the same as cutting the window)
// and builds level L from level L - 1 in shared memory, max of (r, c), (r, c + h), (r + h, c), (r + h, c + h), h = 2^(L-1).
constexpr int kWinTile = 32, kWinSpan = kWinTile + (1 << kPyrLevels) - 1;   // 63
__global__ void __launch_bounds__(256) scan_window_max_kernel(const uint32_t* __restrict__ scan_rimg, int rows, int cols, float empty_value,
                                                              unsigned pyr_stride, float* __restrict__ pyr) {
    __shared__ float buf[2][kWinSpan][kWinSpan + 1];
    const int k = blockIdx.z, r0 = blockIdx.y * kWinTile, c0 = blockIdx.x * kWinTile, npx = rows * cols;
    const uint32_t* img = scan_rimg + (size_t)k * npx;
    const float ninf = -__int_as_float(0x7f800000);
    for (int e = threadIdx.x; e < kWinSpan * kWinSpan; e += blockDim.x) {
        const int y = e / kWinSpan, x = e - y * kWinSpan, r = r0 + y, c = c0 + x;
        float v = ninf;
        if (r < rows && c < cols) { const uint32_t b = img[r * cols + c]; v = (b == 0x461C4000u) ? empty_value : __uint_as_float(b); }
        buf[0][y][x] = v;
    }
    __syncthreads();
    float* out = pyr + (size_t)k * pyr_stride;
    int span = kWinSpan;
    for (int L = 1; L <= kPyrLevels; ++L) {
        const int h = 1 << (L - 1), src = (L - 1) & 1;
        span -= h;                                   // level L is needed over (32 + 2^5 - 2^L)^2 pixels
        for (int e = threadIdx.x; e < span * span; e += blockDim.x) {
            const int y = e / span, x = e - y * span;
            const float m = fmaxf(fmaxf(buf[src][y][x], buf[src][y][x + h]), fmaxf(buf[src][y + h][x], buf[src][y + h][x + h]));
            buf[src ^ 1][y][x] = m;
            const int r = r0 + y, c = c0 + x;
            if (y < kWinTile && x < kWinTile && r < rows && c < cols) out[(size_t)(L - 1) * npx + r * cols + c] = m;
        }
        __syncthreads();
    }
}

// true iff no point of the tile can be a candidate in keyframe k (kf = its fast constants).  Every comparison is written so
// that NaN / degenerate geometry yields "false" (keep the tile).
// kAdaptive (`thres` = c, pixel threshold t = fl(c s)): a pair is a candidate only if s - rho > t (fl(s - rho) > t for a float t).
// Round to nearest gives t >= c s (1 - u), u = 2^-24, so s - t <= s (1 - c (1 - u)), which is non-decreasing in s (c < 1): every pixel
// of the rectangle has s - t <= smax (1 - c (1 - u)).  With c' = fl_down(c (1 - u)) <= c (1 - u) and k1 = fl_up(1 - c') >= 1 - c (1 - u):
//     fl_up(smax k1) <= fl_down(rmin - 1 mm)   =>   s - t <= smax k1 <= rmin - 1 mm < rho   for every point of the tile,
// so no pair is a candidate.  The window table of s is the one of the constant threshold.
template <bool kAdaptive = false>
LTR_DEV bool tile_culled(const float* __restrict__ kf, float4 tile, const FastCfg& fc, const ImgShape& g, const CullArgs& ca, int k, float thres) {
    if (kf[15] == 0.0f) return false;
    const FastProj f = fast_project(kf, tile.x, tile.y, tile.z);   // f.r = |c - o|, f.rho_inv_r = 1 / cos(elevation of c)
    const float d = f.r;
    const float x = __fmul_rn(__fmul_rn(tile.w, mufu_rcp(d)), 1.00001f);     // sin(theta) = rho / d
    const float y = __fmul_rn(x, f.rho_inv_r);                                 // sin(theta) / cos(el_c) bounds sin(azimuth half-width)
    if (!(x <= 0.5f) || !(y <= 0.5f)) return false;                           // asin(t) <= 1.05 t on [0, 0.5]; the cone must not contain the pole
    const float vcol = __fmaf_rn(f.az, fc.col_scale, fc.col_off);
    const float vrow = __fmaf_rn(-f.el, fc.row_scale, fc.row_off);
    const float dc = __fmaf_rn(__fmul_rn(1.05f, y), fc.col_scale, 1.5f);       // half-widths in pixels (+1.5 px: rounding, approximation)
    const float dr = __fmaf_rn(__fmul_rn(1.05f, x), fc.row_scale, 1.5f);
    const float c0f = floorf(__fsub_rn(vcol, dc)), c1f = ceilf(__fadd_rn(vcol, dc));
    if (!(c0f >= 0.0f) || !(c1f <= (float)(g.cols - 1))) return false;         // azimuth seam (or NaN): keep
    if (!(vrow == vrow) || !(dr == dr)) return false;
    const int c0 = (int)c0f, c1 = (int)c1f;
    const int r0 = min(max((int)fminf(fmaxf(floorf(__fsub_rn(vrow, dr)), -1.0f), 1.0e6f), 0), g.rows - 1);  // rows clamp exactly like the pixel index does
    const int r1 = min(max((int)fminf(fmaxf(ceilf(__fadd_rn(vrow, dr)), -1.0f), 1.0e6f), 0), g.rows - 1);
    // cover the rectangle with windows of side s = 2^L: s <= its shorter side where possible (no window reaches beyond it), s >= a quarter of
    // its longer side (at most 4 x 4 windows, 2 x 2 for a near-square rectangle); a side shorter than s gets one window, which reaches
    // beyond the rectangle -- a larger set, still sound
    const int hgt = r1 - r0 + 1, wid = c1 - c0 + 1, lo = min(hgt, wid), hi = max(hgt, wid);
    if (hi > 64) return false;
    int L = max(31 - __clz(lo), 30 - __clz(hi - 1));                             // max(floor(log2(lo)), ceil(log2(hi)) - 2)
    L = min(max(L, 1), kPyrLevels);
    const int s = 1 << L;
    const float* P = ca.pyr + (size_t)k * ca.pyr_stride + (size_t)(L - 1) * (g.rows * g.cols);
    float smax = -__int_as_float(0x7f800000);
    for (int r = r0;; r += s) {
        const int rr = (r + s - 1 >= r1) ? max(min(r, r1 - s + 1), r0) : r;     // the last window ends at r1 (or starts at r0 when s > hgt)
        for (int c = c0;; c += s) {
            const int cc = (c + s - 1 >= c1) ? max(min(c, c1 - s + 1), c0) : c;
            smax = fmaxf(smax, P[rr * g.cols + cc]);
            if (c + s - 1 >= c1) break;
        }
        if (r + s - 1 >= r1) break;
    }
    const float rmin = __fsub_rn(__fsub_rn(__fmul_rn(d, 0.999996f), tile.w), 1.0e-4f);
    if (kAdaptive) {
        const float k1 = __fsub_ru(1.0f, __fmul_rd(thres, 0.99999994f));        // 0.99999994f == 1 - 2^-24 exactly
        return __fmul_ru(smax, k1) <= __fsub_rd(rmin, 1.0e-3f);
    }
    return smax <= __fsub_rn(__fadd_rn(rmin, thres), 1.0e-3f);                 // scan - range <= thres - 1 mm for every point of the tile
}

}  // namespace ltr
