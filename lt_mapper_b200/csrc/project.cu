// libltr_b200.so -- range-image projection kernels: remove / revert / ND / PD pass and visible-point extraction.
//
// Reference functions replaced (paths relative to the lt-mapper repository):
//   Removerter::scan2RangeImg                                   ltremovert/src/Removerter.cpp:109-156
//   transformGlobalMapToLocal + map2RangeImg                    ltremovert/src/utility.cpp:64-72, 92-142
//   range diff + calcDescrepancyAndParseDynamicPointIdx         ltremovert/src/Removerter.cpp:572/459/516, 381-413
//   calcDescrepancyAndParseDynamicPointIdxForEachScan{,ND,PD}   ltremovert/src/Removerter.cpp:542-593, 485-540, 429-482
//   parseProjectedPoints / Session::parseScansViaProjection     ltremovert/src/utility.cpp:74-89, ltremovert/src/Session.cpp:348-360
//
// Determinism: the reference's per-pixel min is a racy OpenMP loop; its sequential meaning (min range, lowest
// index among equal ranges) is obtained here with one 64-bit atomicMin on (float_bits(range) << 32 | index).
#include "ltr_internal.cuh"
#include "device_util.cuh"
#include "ref_math.cuh"
#include "project_fast.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <tuple>
#include <type_traits>

namespace ltr {

constexpr uint32_t kNoPointBits = 0x461C4000u;                       // 10000.0f == kFlagNoPOINT (utility.h:93)
constexpr uint64_t kWinEmpty = ((uint64_t)kNoPointBits << 32);        // (range 10000, index 0) == utility.cpp:103-104
constexpr uint64_t kWinNone = ~0ull;                                  // "no candidate" for the scan-minus-map variants
constexpr float kValidDiffUpperBound = 200.0f;                        // utility.h:94

__global__ void fill_u32_kernel(uint32_t* __restrict__ p, uint32_t v, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void fill_u64_kernel(uint64_t* __restrict__ p, uint64_t v, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// scan2RangeImg for the keyframes [kf0, kf0+nb): per-pixel min range via 32-bit atomicMin on the float bits (ranges >= 0).
__global__ void __launch_bounds__(256) scan_rimg_kernel(PtrView scans, const int64_t* __restrict__ off, int kf0, int nb, ImgShape g,
                                                        uint32_t* __restrict__ rimg) {
    const int64_t begin = off[kf0], end = off[kf0 + nb];
    const int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= end) return;
    const int k = find_kf(off + kf0, nb, i);
    const Sph s = cart2sph(scans.x[i], scans.y[i], scans.z[i]);
    int r, c;
    pixel_index(s, g, &r, &c);
    atomicMin(&rimg[(size_t)k * g.rows * g.cols + (size_t)r * g.cols + c], __float_as_uint(s.r));
}

// The same image through the fast pixel evaluation of project_fast.cuh.  Scan points are already in the sensor frame, so only the
// angle polynomials are approximate; the column / row are accepted when every value within the margins (the ones validated for the map
// projection, which additionally cover a transform error that does not exist here) rounds to the same pixel, otherwise -- pixel
// boundary, point on the z axis -- the reference arithmetic decides.  The range written is always the exact one.
template <bool kElDirect>
__global__ void __launch_bounds__(256) scan_rimg_fast_kernel(PtrView scans, const int64_t* __restrict__ off, int kf0, int nb, ImgShape g, FastCfg fc,
                                                             uint32_t* __restrict__ rimg) {
    const int64_t begin = off[kf0], end = off[kf0 + nb];
    const int64_t i = begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= end) return;
    const int k = find_kf(off + kf0, nb, i);
    const float x = scans.x[i], y = scans.y[i], z = scans.z[i];
    const FastProj f = fast_sph<kElDirect>(x, y, z);
    int r, c;
    const bool okc = certain_round(__fmaf_rn(f.az, fc.col_scale, fc.col_off), __fmaf_rn(fc.m_col_b, f.rho_inv_r, fc.m_col_a), g.cols - 1, &c);
    const bool okr = certain_round(__fmaf_rn(f.el, fc.neg_row_scale, fc.row_off), fc.m_row, g.rows - 1, &r);
    float range;
    if (okc & okr) {
        range = __fsqrt_rn(fa(fa(fm(x, x), fm(y, y)), fm(z, z)));   // cart2sph's r (utility.cpp:48)
    } else {
        const Sph s = cart2sph(x, y, z);
        pixel_index(s, g, &r, &c);
        range = s.r;
    }
    atomicMin(&rimg[(size_t)k * g.rows * g.cols + (size_t)r * g.cols + c], __float_as_uint(range));
}

// test image of the scan-minus-map fast path (project_fast.cuh) for nb keyframes: the scan image, with "no return" pixels set to -inf when
// `empty_to_ninf` (that makes "scan - range > thres" false for every range -- valid when no map point can be ~10000 m away,
// empty_scan_shortcut_ok).  With pad_g guard rows above and below and pad_c = 1 guard column (FastCfg::pad_*) the guard rows replicate the
// rows that pixel_index clamps to, so the short elevation path gathers from it without clamping its index, and column 0 and the guard column
// hold +inf: the pixels next to the azimuth seam, whose pairs map_project_fast_kernel sends to the full exact path.  pad_g = pad_c = 0: plain layout.
// kAdaptive (pixel threshold fl(c s), Removerter.cpp:396): every other pixel holds fl_up(s - fl(c s)) instead of s -- an upper bound of
// s - t that the fast kernel tests against 0 (project_fast.cuh); a pixel without a return too, unless the shortcut made it -inf.
template <bool kAdaptive = false>
__global__ void __launch_bounds__(256) scan_test_image_kernel(const uint32_t* __restrict__ rimg, uint32_t* __restrict__ test_img, int nb, int rows, int cols,
                                                              int pad_g, int pad_c, int empty_to_ninf, float coeff) {
    const int W = cols + pad_c;
    const int64_t per_kf = (int64_t)(rows + 2 * pad_g) * W, n = nb * per_kf;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(i / per_kf);
        const int p = (int)(i - k * per_kf);
        const int rp = p / W;
        const int cp = p - rp * W;
        const int r = min(max(rp - pad_g, 0), rows - 1), c = min(cp, cols - 1);
        const uint32_t b = rimg[(size_t)k * rows * cols + (size_t)r * cols + c];
        const uint32_t v = kAdaptive ? __float_as_uint(__fsub_ru(__uint_as_float(b), fm(coeff, __uint_as_float(b)))) : b;
        test_img[i] = (pad_c && (cp == 0 || cp == cols)) ? 0x7f800000u : (empty_to_ninf && b == kNoPointBits) ? 0xff800000u : v;
    }
}

// Exact projection of every map point into every keyframe of the batch.
//   kCandidatesOnly = true  (HD / revert / PD, diff = scan - map): by monotonicity of f32 subtraction the set
//       {points with scan - range > t} is a prefix in range order of the pixel's points, so the pixel winner among
//       them equals the global pixel winner whenever any exists; only those points touch the atomic (SURVEY.md §A.2).
//       The argument needs t constant within a pixel, not across pixels: it holds for the adaptive t = fl(c s) (kAdaptive,
//       `thres` = c), which only depends on the pixel's scan range s.
//   kCandidatesOnly = false (ND, visible-point extraction): true per-pixel minimum with a read-before-atomic filter.
//   kBall: keyframe k of the launch sees only the points of its ball (ball_member with ball_c[k], ball_r2), every pair tested.
template <bool kCandidatesOnly, bool kAdaptive = false, bool kBall = false>
__global__ void __launch_bounds__(256) map_project_kernel(PtrView map, const double* __restrict__ poses, int kf0, int nb,
                                                          const double* __restrict__ ext, int ext_identity, int order, ImgShape g,
                                                          const uint32_t* __restrict__ scan_rimg, float thres, uint64_t* __restrict__ win,
                                                          const float4* __restrict__ ball_c, float ball_r2) {
    extern __shared__ double s_pose[];  // nb * 12: inverse poses of the batch
    for (int t = threadIdx.x; t < nb * 12; t += blockDim.x) s_pose[t] = poses[(size_t)(kf0 + t / 12) * 24 + (t % 12)];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= map.n) return;
    const float x = map.x[i], y = map.y[i], z = map.z[i];
    unsigned n_atomics = 0;   // not reported by this kernel
    for (int k = 0; k < nb; ++k) {
        if (kBall && !ball_member(x, y, z, ball_c[k], ball_r2)) continue;
        exact_pair<kCandidatesOnly, kAdaptive>(x, y, z, (uint32_t)i, (uint32_t)k, s_pose + 12 * k, ext, ext_identity, order, g, scan_rimg, thres, win, 0, &n_atomics);
    }
}

// calcDescrepancyAndParseDynamicPointIdx (Removerter.cpp:381-413) over the batch images; also re-arms `win`.  kAdaptive: the threshold
// is fl(c s) of the pixel's scan range s (Removerter.cpp:396 in place of :398), c in `thres`.
template <bool kCandidatesOnly, bool kAdaptive = false>
__global__ void __launch_bounds__(256) resolve_kernel(const uint32_t* __restrict__ scan_rimg, uint64_t* __restrict__ win, int64_t total_px,
                                                      float thres, uint8_t* __restrict__ flags) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= total_px) return;
    const uint64_t w = win[p];
    if (kCandidatesOnly) {
        if (w == kWinNone) return;
        win[p] = kWinNone;
        const float mr = __uint_as_float((uint32_t)(w >> 32)), sr = __uint_as_float(scan_rimg[p]);
        const float diff = fs(sr, mr);  // scan - map (Removerter.cpp:572, 459)
        if (diff < kValidDiffUpperBound && diff > pixel_thres<kAdaptive>(thres, sr)) flags[(uint32_t)w] = 1;
    } else {
        if (w != kWinEmpty) win[p] = kWinEmpty;
        const float mr = __uint_as_float((uint32_t)(w >> 32)), sr = __uint_as_float(scan_rimg[p]);
        const float diff = fs(mr, sr);  // map - scan (Removerter.cpp:516)
        if (diff < kValidDiffUpperBound && diff > pixel_thres<kAdaptive>(thres, sr)) flags[(uint32_t)w] = 1;
    }
}

// parseProjectedPoints (utility.cpp:80-87): row-major scan of the index image, skipping index 0.  Each keyframe's image is cut
// into chunks of kParseChunk pixels, one block per (chunk, keyframe): a count kernel, then a scatter kernel that starts at the sum of
// the preceding chunks' counts and compacts its chunk in pixel order (and resets the winner image for the next batch).
constexpr int kParseChunk = 8192;

__global__ void __launch_bounds__(1024) parse_count_kernel(const uint64_t* __restrict__ win, int npx, int nchunk, unsigned int* __restrict__ chunk_cnt) {
    __shared__ int s_warp[32];
    const int k = blockIdx.y, c = blockIdx.x;
    const uint64_t* w = win + (size_t)k * npx;
    const int p1 = min((c + 1) * kParseChunk, npx);
    int n = 0;
    for (int p = c * kParseChunk + threadIdx.x; p < p1; p += blockDim.x) n += ((uint32_t)w[p] != 0u) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x < 32) {
        n = s_warp[threadIdx.x];
        for (int o = 16; o > 0; o >>= 1) n += __shfl_down_sync(0xffffffffu, n, o);
        if (threadIdx.x == 0) chunk_cnt[(size_t)k * nchunk + c] = (unsigned int)n;
    }
}

__global__ void __launch_bounds__(1024) parse_compact_kernel(uint64_t* __restrict__ win, int npx, int nchunk, const unsigned int* __restrict__ chunk_cnt,
                                                             uint32_t* __restrict__ list, unsigned int* __restrict__ count) {
    __shared__ int s_warp[33];
    __shared__ int s_base;
    const int k = blockIdx.y, c = blockIdx.x;
    uint64_t* w = win + (size_t)k * npx;
    uint32_t* out = list + (size_t)k * npx;
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp == 0) {   // where this chunk's output starts: the counts of the chunks before it
        int b = 0;
        for (int j = (int)lane; j < c; j += 32) b += (int)chunk_cnt[(size_t)k * nchunk + j];
        for (int o = 16; o > 0; o >>= 1) b += __shfl_down_sync(0xffffffffu, b, o);
        if (lane == 0) s_base = b;
    }
    __syncthreads();
    int base = s_base;
    const int p1 = min((c + 1) * kParseChunk, npx);
    for (int p0 = c * kParseChunk; p0 < p1; p0 += blockDim.x) {
        const int p = p0 + threadIdx.x;
        uint32_t idx = 0;
        if (p < p1) { const uint64_t v = w[p]; idx = (uint32_t)v; if (v != kWinEmpty) w[p] = kWinEmpty; }
        int total;
        const int rank = block_rank(idx != 0, &total, s_warp);
        if (idx != 0) out[base + rank] = idx;
        base += total;
    }
    if (c == nchunk - 1 && threadIdx.x == 0) count[k] = (unsigned int)base;
}

// emits map_local[ptidx] for every listed index: exact two-step transform of the winning map point
__global__ void __launch_bounds__(256) parse_emit_kernel(PtrView map, const double* __restrict__ poses, int kf_begin, const int64_t* __restrict__ out_off,
                                                         int K, const uint32_t* __restrict__ list, int npx, const double* __restrict__ ext,
                                                         int ext_identity, int order, DevCloud out) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= out.n) return;
    const int k = find_kf(out_off, K, j);
    const uint32_t idx = list[(size_t)k * npx + (size_t)(j - out_off[k])];
    float x, y, z;
    map_to_sensor(poses + (size_t)(kf_begin + k) * 24, ext, ext_identity, order, map.x[idx], map.y[idx], map.z[idx], &x, &y, &z);
    out.x()[j] = x; out.y()[j] = y; out.z()[j] = z; out.i()[j] = map.i[idx];
}

__global__ void debug_pixel_kernel(const float* __restrict__ xyz, int64_t n, ImgShape g, int* __restrict__ row, int* __restrict__ col,
                                   float* __restrict__ range, float* __restrict__ az, float* __restrict__ el) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Sph s = cart2sph(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    int r, c;
    pixel_index(s, g, &r, &c);
    row[i] = r; col[i] = c; range[i] = s.r; az[i] = s.az; el[i] = s.el;
}

// records an event pair around the dominant kernel; collected by prof_collect after the pass's final synchronisation
static inline void prof_begin(ltr_ctx* ctx) { if (ctx->ev_used + 2 <= (int)ctx->ev_pool.size()) cudaEventRecord(ctx->ev_pool[ctx->ev_used], ctx->stream); }
static inline void prof_end(ltr_ctx* ctx) { if (ctx->ev_used + 2 <= (int)ctx->ev_pool.size()) { cudaEventRecord(ctx->ev_pool[ctx->ev_used + 1], ctx->stream); ctx->ev_used += 2; } }
static inline void prof_collect(ltr_ctx* ctx, int slot, double bytes_per_launch_unit, double proj_per_launch_unit, const std::vector<int>& units) {
    // units[i] = keyframes in launch i (only the launches that got an event pair are accumulated)
    for (int i = 0; i * 2 + 1 < ctx->ev_used && i < (int)units.size(); ++i) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, ctx->ev_pool[2 * i], ctx->ev_pool[2 * i + 1]) != cudaSuccess) continue;
        ctx->prof[slot + 0] += (double)ms * 1000.0;
        ctx->prof[slot + 1] += 1.0;
        ctx->prof[slot + 2] += bytes_per_launch_unit * units[i];
        ctx->prof[slot + 3] += proj_per_launch_unit * units[i];
    }
    ctx->ev_used = 0;
}

// 1 iff no map point can be >= 8000 m away from any keyframe origin in [k0, k1): then a pixel without a scan return
// (scan range 10000) has scan - map > 200 for every map point and can never flag (see project_fast.cuh).
static int empty_scan_shortcut_ok(ltr_ctx* ctx, const DevCloud& map, const DevPoses& poses, int k0, int k1, int* ok) {
    *ok = 0;
    float mn[3], mx[3];
    LTR_TRY(minmax_xyz(ctx, map, mn, mx));
    double worst = 0.0;
    for (int k = k0; k < k1; ++k) {
        const float* f = &poses.h_fast[(size_t)k * 16];
        if (f[15] == 0.0f) return LTR_OK;
        double d2 = 0.0;
        for (int d = 0; d < 3; ++d) {
            const double c = (double)f[9 + d];  // c_hi (the f32 part of the sensor origin is plenty for a 7 km bound)
            const double e = std::max(std::fabs(c - (double)mn[d]), std::fabs(c - (double)mx[d]));
            d2 += e * e;
        }
        worst = std::max(worst, d2);
    }
    *ok = (worst < 7000.0 * 7000.0) ? 1 : 0;
    return LTR_OK;
}

template <bool kElDirect>
__global__ void debug_fast_kernel(const float* __restrict__ xyz, int64_t n, const float* __restrict__ kf, const double* __restrict__ pose,
                                  const double* __restrict__ ext, int ext_identity, int order, ImgShape g, FastCfg fc,
                                  float* __restrict__ out /* n x 8: vcol_f vrow_f r_f rho_inv_r | vcol_e vrow_e r_e az_f */) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const FastProj f = fast_project<kElDirect>(kf, x, y, z);
    out[8 * i + 0] = __fmaf_rn(f.az, fc.col_scale, fc.col_off);
    out[8 * i + 1] = __fmaf_rn(f.el, fc.neg_row_scale, fc.row_off);
    out[8 * i + 2] = f.r;
    out[8 * i + 3] = f.rho_inv_r;
    float lx, ly, lz;
    map_to_sensor(pose, ext, ext_identity, order, x, y, z, &lx, &ly, &lz);
    const Sph s = cart2sph(lx, ly, lz);
    // the reference's pre-round floats (utility.cpp:122-123)
    out[8 * i + 4] = fm((float)g.cols, fd(fa(rad2deg(s.az), fd(g.hfov, 2.0f)), fs(g.hfov, 0.0f)));
    out[8 * i + 5] = fm((float)g.rows, fs(1.0f, fd(fa(rad2deg(s.el), fd(g.vfov, 2.0f)), fs(g.vfov, 0.0f))));
    out[8 * i + 6] = s.r;
    out[8 * i + 7] = f.az;   // the fast azimuth, for the seam rule of map_project_fast_kernel
}

// Exhaustive check of the two arctangent polynomials of the fast path: every float a with bits in [0, last_bits] (i.e. all of [0, 1]
// or [0, 0.5]) is evaluated and compared with atan((double)a); the maximum absolute error is kept (positive doubles order like their bits).
__global__ void __launch_bounds__(256) atan_sweep_kernel(int which, uint32_t last_bits, unsigned long long* __restrict__ max_err_bits, uint32_t* __restrict__ arg_bits) {
    double worst = 0.0;
    uint32_t worst_arg = 0;
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b <= last_bits; b += (uint64_t)gridDim.x * blockDim.x) {
        const float a = __uint_as_float((uint32_t)b);
        const float v = which == 0 ? fast_atan01(a) : fast_atan_half(a);
        const double e = fabs((double)v - atan((double)a));
        if (e > worst) { worst = e; worst_arg = (uint32_t)b; }
    }
    const unsigned long long wb = (unsigned long long)__double_as_longlong(worst);
    const unsigned long long old = atomicMax(max_err_bits, wb);
    if (wb > old) *arg_bits = worst_arg;   // racy between equal-ish maxima; the argument is informational only
}

// the 128-point tiles of a map of n points: the work units of map_project_fast_kernel's warps, and what culling, the ball and the
// near-to-far claim order bound with a sphere
static inline long long tile_count(int64_t n) { return (n + kTilePts - 1) / kTilePts; }

// the bounding spheres of the map's tiles (float4 per tile) into a new scratch block *spheres; a pass computes them once for all readers
static int tile_spheres(ltr_ctx* ctx, const DevCloud& map, void** spheres) {
    const long long ntiles = tile_count(map.n);
    LTR_TRY(dev_alloc(ctx, spheres, (size_t)ntiles * sizeof(float4)));
    tile_sphere_kernel<<<(unsigned)((ntiles * 32 + 255) / 256), 256, 0, ctx->stream>>>(view(map), (float4*)*spheres, ntiles);
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

// persistent grid: up to 4 resident CTAs per SM (20 KB shared memory each; the 3-CTA variants leave the rest queued: the warps claim tiles
// from a counter, so a late CTA only finds less work), never more CTAs than tiles need
static inline unsigned fast_grid(const ltr_ctx* ctx, int64_t n) {
    const int64_t ctas = (tile_count(n) + kFastThreads / 32 - 1) / (kFastThreads / 32);
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ctas, (int64_t)ctx->sm_count * kFastCtasPerSmPad));
}

static inline size_t fast_smem_bytes() { return (size_t)(kFastThreads / 32) * 2 * kQueueCap * sizeof(uint64_t); }

static inline unsigned grid_for(int64_t n, int threads, int max_blocks) {
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads, max_blocks));
}

static inline KfBatch make_kf_batch(const DevPoses& poses, int k0, int nb) {
    KfBatch kb;
    std::memset(&kb, 0, sizeof(kb));
    std::memcpy(kb.kf, &poses.h_fast[(size_t)k0 * 16], (size_t)nb * 16 * sizeof(float));
    return kb;
}

// What a pass resolves once per call.
struct PassPlan {
    ImgShape g;
    int64_t npx;
    bool use_fast;           // the fast path, within its queue-entry field widths and 32-bit pixel offsets (project_fast.cuh)
    FastCfg fc;              // its constants; empty_scan_shortcut = 0 until the remove pass sets its own
    int B;                   // keyframes per launch: fast path at most kFastMaxBatch (their constants travel as a kernel parameter), exact
                             // path 12 doubles of shared memory per keyframe
    std::vector<int> units;  // keyframes of each projection launch (prof_collect)
};

static int plan_pass(ltr_ctx* ctx, float res_alpha, int nkf, PassPlan* p) {
    int32_t rows, cols;
    ltr_reset_rimg_size(ctx->cfg.vfov_deg, ctx->cfg.hfov_deg, res_alpha, &rows, &cols);
    if (rows < 1 || cols < 1) return fail(ctx, LTR_ERR_INVALID, "range image %dx%d is empty (res_alpha %g)", rows, cols, res_alpha);
    p->g = ImgShape{rows, cols, ctx->cfg.vfov_deg, ctx->cfg.hfov_deg};
    p->npx = (int64_t)rows * cols;
    p->use_fast = ctx->cfg.fast_path && p->npx <= (1 << 18);
    p->fc = make_fast_cfg(rows, cols, ctx->cfg.vfov_deg, ctx->cfg.hfov_deg, 0);
    p->B = std::max(1, std::min(std::min(ctx->cfg.keyframe_batch, p->use_fast ? kFastMaxBatch : 400), nkf));
    return LTR_OK;
}

// the keyframe range of a pass over K keyframes, and a map whose indices fit the 32-bit index half of the winner image's keys
static int check_pass_range(ltr_ctx* ctx, const DevCloud& map, int kf_begin, int kf_end, int K) {
    if (kf_begin < 0 || kf_end > K || kf_begin > kf_end) return fail(ctx, LTR_ERR_INVALID, "keyframe range [%d,%d) outside [0,%d)", kf_begin, kf_end, K);
    if (map.n >= ((int64_t)1 << 32)) return fail(ctx, LTR_ERR_UNSUPPORTED, "map larger than 2^32 points");
    return LTR_OK;
}

// start of a pass's timed part: the fast path's device counters, the start event, no event pairs yet
static int pass_begin(ltr_ctx* ctx, const PassPlan& p) {
    if (p.use_fast) LTR_CUDA(ctx, cudaMemsetAsync(ctx->d_counters, 0, 4 * sizeof(unsigned long long), ctx->stream));
    LTR_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
    ctx->ev_used = 0;
    return LTR_OK;
}

// after the pass's final synchronisation on ev1: the projection launches' event pairs into prof[slot .. slot + 3], and stats[0..4] of a
// pass over n map points and nkf keyframes (the fast path's device counters are fetched lazily by ltr_last_pass_stats)
static void pass_end(ltr_ctx* ctx, const PassPlan& p, int slot, double bytes_per_launch_unit, int64_t n, int nkf) {
    float ms = 0.0f;
    cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    prof_collect(ctx, slot, bytes_per_launch_unit, (double)n, p.units);
    ctx->stats[0] = (double)n * nkf;
    ctx->stats[1] = 0; ctx->stats[2] = ctx->stats[0]; ctx->stats[3] = 0;
    ctx->stats_counters_pending = p.use_fast;
    ctx->stats[4] = (double)ms * 1000.0;
}

// Runtime bools as template arguments: with_bools(f, a, b) returns f(std::bool_constant<a>{}, std::bool_constant<b>{}).  f is
// instantiated for every combination, so it must name only the kernels it may be asked for.
template <class F>
static auto with_bools(F f) { return f(); }
template <class F, class... Rest>
static auto with_bools(F f, bool b, Rest... rest) {
    const auto bind = [&](auto c) { return with_bools([&](auto... cs) { return f(c, cs...); }, rest...); };
    return b ? bind(std::true_type{}) : bind(std::false_type{});
}

// what one launch of the map projection computes in the winner image
enum class Proj {
    kScanMinusMap,      // HD / revert / PD: the pixel winner among the candidates, scan - map > thres
    kTrueMin,           // ND, visible-point extraction: the true per-pixel minimum
    kTrueMinDeferred,   // the same through the deferred mode of project_fast.cuh (fast path only): the fast kernel, then deferred_resolve_kernel
};

// One launch of the map projection over the keyframes [k0, k0 + nb) of `poses` into `win`, timed by an event pair.  rimg: the launch's scan
// range images (scan-minus-map; unused by the true minimum), test_img: the test image of the scan-minus-map fast path.  amin (fast path,
// may be null in the deferred mode): the approximate running minimum, reset here.  da: the deferred mode's scratch.  adaptive (scan-minus-map
// only): `thres` is the coefficient c of the pixel threshold fl(c s), and test_img was built for it.  ball (args.centre nullptr: the full
// map): keyframe k sees only the points of its ball (args.centre[k], args.r2); on the fast path through the tile list of the
// launch, which ball_tile_list_kernel builds here from the tile spheres and non-finite flags into `scratch` (3 ntiles words: out masks,
// in masks, list).
struct BallLaunch {
    BallArgs args{};                   // centre and r2 set by ball_setup, centre moved to each launch's keyframes; the rest by project_map
    const float4* tiles = nullptr;
    const uint8_t* nonfinite = nullptr;
    long long ntiles = 0;
    uint32_t* scratch = nullptr;
    std::vector<float4> h_centre;      // host copy of the centres: outlives their upload, the pass synchronises before it returns
};

static int project_map(ltr_ctx* ctx, PassPlan& p, const DevCloud& map, const DevPoses& poses, int k0, int nb, Proj mode, const uint32_t* rimg,
                       const uint32_t* test_img, float thres, bool adaptive, uint64_t* win, uint32_t* amin, const CullArgs& ca, const DeferredArgs& da,
                       const BallLaunch& ball = BallLaunch{}) {
    const bool cand = mode == Proj::kScanMinusMap;
    adaptive = adaptive && cand;
    const bool use_ball = ball.args.centre != nullptr;
    if (amin) {
        fill_u32_kernel<<<grid_for(nb * p.npx, 256, ctx->sm_count * 8), 256, 0, ctx->stream>>>(amin, 0x7f800000u, nb * p.npx);
        LTR_LAUNCH_CHECK(ctx);
    }
    prof_begin(ctx);
    p.units.push_back(nb);
    if (!p.use_fast) {
        const auto kern = with_bools([cand](auto ad, auto in_ball) {
            return cand ? map_project_kernel<true, ad, in_ball> : map_project_kernel<false, false, in_ball>;
        }, adaptive, use_ball);
        kern<<<(unsigned)((map.n + 255) / 256), 256, (size_t)nb * 12 * sizeof(double), ctx->stream>>>(view(map), poses.d, k0, nb, ctx->d_ext,
            ctx->ext_identity ? 1 : 0, ctx->cfg.transform_order, p.g, rimg, thres, win, ball.args.centre, ball.args.r2);
    } else {
        unsigned int* work = (unsigned int*)(ctx->d_counters + 4);
        LTR_CUDA(ctx, cudaMemsetAsync(work, 0, sizeof(unsigned int), ctx->stream));
        const bool deferred = mode == Proj::kTrueMinDeferred;
        if (deferred) {
            LTR_CUDA(ctx, cudaMemsetAsync(da.best, 0xff, (size_t)nb * p.npx * sizeof(unsigned long long), ctx->stream));   // "no pair yet"
            LTR_CUDA(ctx, cudaMemsetAsync(da.count, 0, sizeof(unsigned int), ctx->stream));
        }
        BallArgs ba{};
        if (use_ball) {   // the launch's tile list; its count lives in counters[5], never read by the host
            ba = ball.args;
            uint32_t* s = ball.scratch;
            unsigned int* count = (unsigned int*)(ctx->d_counters + 5);
            ba.out_mask = s; ba.in_mask = s + ball.ntiles; ba.list = s + 2 * ball.ntiles; ba.count = count;
            LTR_CUDA(ctx, cudaMemsetAsync(count, 0, sizeof(unsigned int), ctx->stream));
            ball_tile_list_kernel<<<(unsigned)((ball.ntiles * 32 + 255) / 256), 256, 0, ctx->stream>>>(ball.tiles, ball.nonfinite, ball.ntiles, ba, nb,
                s, s + ball.ntiles, s + 2 * ball.ntiles, count, ctx->d_counters);
            LTR_LAUNCH_CHECK(ctx);
        }
        // template arguments <candidates only, short elevation path, deferred, guard-padded test image, adaptive threshold, ball subset>;
        // the padded test image implies the short elevation path (FastCfg::pad_ok)
        const auto kern = with_bools([mode, pad = cand && p.fc.pad_ok](auto el, auto ad, auto in_ball) {
            return pad                         ? map_project_fast_kernel<true, true, false, true, ad, in_ball>
                 : mode == Proj::kScanMinusMap ? map_project_fast_kernel<true, el, false, false, ad, in_ball>
                 : mode == Proj::kTrueMin      ? map_project_fast_kernel<false, el, false, false, false, in_ball>
                                               : map_project_fast_kernel<false, el, true, false, false, in_ball>;
        }, p.fc.el_direct != 0, adaptive, use_ball);
        kern<<<fast_grid(ctx, map.n), kFastThreads, fast_smem_bytes(), ctx->stream>>>(view(map), make_kf_batch(poses, k0, nb), poses.d, k0, nb, ctx->d_ext,
            ctx->ext_identity ? 1 : 0, ctx->cfg.transform_order, p.g, p.fc, rimg, cand ? test_img : amin, thres, win, amin, ca, ctx->d_counters, work, da, ba);
        if (deferred) {
            LTR_LAUNCH_CHECK(ctx);
            deferred_resolve_kernel<<<grid_for(nb * p.npx, 256, ctx->sm_count * 16), 256, 0, ctx->stream>>>(view(map), poses.d, k0, nb, ctx->d_ext,
                ctx->ext_identity ? 1 : 0, ctx->cfg.transform_order, (uint32_t)p.npx, da, win, ctx->d_counters);
        }
    }
    prof_end(ctx);
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

// Fills `bl` with the balls of radius `radius` around the keyframes [kf_begin, kf_end): their f32 centres and, on the fast path, the pass's
// tile spheres, a non-finite flag per tile and the launches' tile-list scratch.  Centres, flags and scratch share one new scratch block
// *block.  PCL's radiusSearch hands FLANN radius^2 as a float; an r2 that rounds to 0 admits no point.
static int ball_setup(ltr_ctx* ctx, const PassPlan& p, const DevCloud& map, const DevPoses& poses, int kf_begin, int kf_end, float radius,
                      const float4* spheres, void** block, BallLaunch* bl) {
    const int K = kf_end - kf_begin;
    const long long ntiles = tile_count(map.n);
    bl->h_centre.resize((size_t)K);
    for (int k = 0; k < K; ++k) {   // the pose's translation column (pose rows at 12..23 of DevPoses::h), rounded to f32
        const double* T = &poses.h[(size_t)(kf_begin + k) * 24 + 12];
        bl->h_centre[(size_t)k] = make_float4((float)T[3], (float)T[7], (float)T[11], 0.0f);
    }
    const size_t c_bytes = ((size_t)K * sizeof(float4) + 255) / 256 * 256;
    const size_t w_bytes = p.use_fast ? ((size_t)ntiles * 3 * sizeof(uint32_t) + 255) / 256 * 256 : 0;
    LTR_TRY(dev_alloc(ctx, block, c_bytes + w_bytes + (p.use_fast ? (size_t)ntiles : 0)));
    char* b = (char*)*block;
    LTR_CUDA(ctx, cudaMemcpyAsync(b, bl->h_centre.data(), (size_t)K * sizeof(float4), cudaMemcpyHostToDevice, ctx->stream));
    bl->args.centre = (const float4*)b;
    bl->args.r2 = (float)((double)radius * (double)radius);
    if (p.use_fast) {
        uint8_t* nonfinite = (uint8_t*)(b + c_bytes + w_bytes);
        LTR_CUDA(ctx, cudaMemsetAsync(nonfinite, 0, (size_t)ntiles, ctx->stream));
        tile_nonfinite_kernel<<<(unsigned)((map.n + 255) / 256), 256, 0, ctx->stream>>>(view(map), nonfinite);
        LTR_LAUNCH_CHECK(ctx);
        bl->tiles = spheres;
        bl->nonfinite = nonfinite;
        bl->ntiles = ntiles;
        bl->scratch = (uint32_t*)(b + c_bytes);
    }
    return LTR_OK;
}

// scan2RangeImg of the keyframes [kf0, kf0 + n) of `scans` into n images at rimg, through the fast pixel evaluation on the fast path
static int scan_rimg(ltr_ctx* ctx, const PassPlan& p, const DevScanSet& scans, int kf0, int n, uint32_t* rimg) {
    fill_u32_kernel<<<grid_for(n * p.npx, 256, ctx->sm_count * 8), 256, 0, ctx->stream>>>(rimg, kNoPointBits, n * p.npx);
    LTR_LAUNCH_CHECK(ctx);
    const int64_t npts = scans.h_off[kf0 + n] - scans.h_off[kf0];
    if (npts == 0) return LTR_OK;
    const unsigned blocks = (unsigned)((npts + 255) / 256);
    if (p.use_fast) {
        const auto kern = with_bools([](auto el) { return scan_rimg_fast_kernel<el>; }, p.fc.el_direct != 0);
        kern<<<blocks, 256, 0, ctx->stream>>>(view(scans.pts), scans.d_off, kf0, n, p.g, p.fc, rimg);
    } else {
        scan_rimg_kernel<<<blocks, 256, 0, ctx->stream>>>(view(scans.pts), scans.d_off, kf0, n, p.g, rimg);
    }
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

// Near-to-far claim order of the deferred mode (DeferredArgs::order): per tile, a lower bound of its distance from `o` (a reference
// origin of the launch's keyframes) quantised to 1/16 m and saturated at 4096 m in key bits 32..47, the tile index in bits 0..31.
// Sorting bits 32..47 (two 8-bit radix passes) keeps equal distances in map order.  The order only changes how fast `best` fills.
constexpr float kOrderSteps = 16.0f;   // per metre
__global__ void __launch_bounds__(256) tile_order_key_kernel(const float4* __restrict__ tiles, long long ntiles, float ox, float oy, float oz,
                                                             uint64_t* __restrict__ keys) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    const float4 s = tiles[t];
    const float dx = s.x - ox, dy = s.y - oy, dz = s.z - oz;
    const float q = fminf(fmaxf((sqrtf(dx * dx + dy * dy + dz * dz) - s.w) * kOrderSteps, 0.0f), 65535.0f);   // NaN -> 0
    keys[t] = ((uint64_t)(uint32_t)q << 32) | (uint64_t)t;
}

// scratch of the deferred true-minimum mode for launches of up to B keyframes: best image + overflow list + its counter
constexpr unsigned kDeferredListCap = 8u << 20;   // entries (64 MB); a typical launch appends a few 10^4
static int deferred_alloc(ltr_ctx* ctx, int B, int64_t npx, void** block, DeferredArgs* da) {
    // Test knob: LTR_DEFERRED_LIST_CAP=n (clamped to kDeferredListCap) shrinks the list the launches may fill, so that tests can make it
    // overflow and exercise the immediate-mode retry of ltr_remove_pass / ltr_parse_projected on small inputs.
    unsigned cap = kDeferredListCap;
    if (const char* e = std::getenv("LTR_DEFERRED_LIST_CAP")) if (*e) cap = (unsigned)std::min<long long>(std::max(std::atoll(e), 0ll), kDeferredListCap);
    const size_t best_bytes = (size_t)B * npx * sizeof(unsigned long long);
    LTR_TRY(dev_alloc(ctx, block, best_bytes + (size_t)kDeferredListCap * sizeof(unsigned long long) + 256));
    da->best = (unsigned long long*)*block;
    da->list = da->best + (size_t)B * npx;
    da->count = (unsigned int*)(da->list + kDeferredListCap);
    da->overflow = da->count + 1;
    da->capacity = cap;
    LTR_CUDA(ctx, cudaMemsetAsync(da->count, 0, 2 * sizeof(unsigned int), ctx->stream));
    return LTR_OK;
}

// Scan-side images of a remove pass for the keyframes [k0, k0 + nb) of `scans`, keyframe-major:
//   rimg  the scan range image (scan2RangeImg), built here when make_rimg, else read;
//   pyr   (if non-null) its sliding-window maxima for tile culling; an empty scan pixel is -inf with the shortcut, else +inf;
//   timg  (if non-null) the test image of the scan-minus-map fast path, guard-padded when `pad`, empty pixels -inf with the shortcut;
//         coeff != 0: the one of the adaptive threshold fl(coeff s) (scan_test_image_kernel).
// The shortcut is the plan's FastCfg::empty_scan_shortcut.  None of them reads the map.  Launches cover at most kImageChunk keyframes (the
// window-maximum grid's z extent).
constexpr int kImageChunk = 1024;
static int build_scan_images(ltr_ctx* ctx, const PassPlan& p, const DevScanSet& scans, int k0, int nb, bool make_rimg, uint32_t* rimg, float* pyr,
                             uint32_t* timg, bool pad, float coeff) {
    const ImgShape& g = p.g;
    const int64_t npx = p.npx;
    const int shortcut = p.fc.empty_scan_shortcut;
    const int64_t timg_px = pad ? (int64_t)p.fc.pad_npx : npx;
    const unsigned pyr_stride = (unsigned)(kPyrLevels * npx);
    const int fill_blocks = ctx->sm_count * 8;
    for (int c0 = 0; c0 < nb; c0 += kImageChunk) {
        const int n = std::min(kImageChunk, nb - c0);
        uint32_t* ri = rimg + (size_t)c0 * npx;
        if (make_rimg) LTR_TRY(scan_rimg(ctx, p, scans, k0 + c0, n, ri));
        if (pyr) {
            const float empty_value = shortcut ? -__builtin_huge_valf() : __builtin_huge_valf();   // empty scan pixel: never flags / unknown
            const dim3 wg((unsigned)((g.cols + kWinTile - 1) / kWinTile), (unsigned)((g.rows + kWinTile - 1) / kWinTile), (unsigned)n);
            scan_window_max_kernel<<<wg, 256, 0, ctx->stream>>>(ri, g.rows, g.cols, empty_value, pyr_stride, pyr + (size_t)c0 * pyr_stride);
            LTR_LAUNCH_CHECK(ctx);
        }
        if (timg) {
            const auto kern = with_bools([](auto ad) { return scan_test_image_kernel<ad>; }, coeff != 0.0f);
            kern<<<grid_for(n * timg_px, 256, fill_blocks), 256, 0, ctx->stream>>>(ri, timg + (size_t)c0 * timg_px, n, g.rows, g.cols, pad ? p.fc.pad_g : 0,
                                                                                  pad ? 1 : 0, shortcut, coeff);
            LTR_LAUNCH_CHECK(ctx);
        }
    }
    return LTR_OK;
}

// Kept scan-image sets (ScanImageSet): the second remove pass at a resolution and the three ND and three PD filter passes find their images.

static void scan_image_set_drop(ScanImageSet& s) {
    s.valid = false;
    s.rimg = nullptr; s.pyr = nullptr; s.timg = nullptr;
    s.pyr_shortcut = s.timg_shortcut = -1;
    s.timg_coeff_bits = 0;
}

void scan_images_release(ltr_ctx* ctx, uint64_t serial, bool free_storage) {
    for (ScanImageSet& s : ctx->scan_images) {
        if (serial == 0 || s.key.scans_serial == serial || s.key.poses_serial == serial) scan_image_set_drop(s);
        if (free_storage && serial == 0) { dev_free(ctx, s.block); s.block = nullptr; s.cap = 0; }
    }
}

bool scan_images_have_storage(const ltr_ctx* ctx) {
    for (const ScanImageSet& s : ctx->scan_images) if (s.block) return true;
    return false;
}

// Bytes the slots' storage may take in all.  LTR_SCAN_IMAGE_CACHE_MB=n sets n MiB; 0 turns the sets off, and every pass builds its images
// per launch.  Default: a quarter of the device memory this context could still use (free, its allocator cache, the slots themselves).
static bool scan_image_cache_on(size_t* fixed_budget) {
    *fixed_budget = 0;
    const char* e = std::getenv("LTR_SCAN_IMAGE_CACHE_MB");
    if (!e || !*e) return true;
    *fixed_budget = (size_t)std::max(std::atoll(e), 0ll) << 20;
    return *fixed_budget > 0;
}

// Pins the slots' storage for the rest of a pass: an allocation that runs out of memory must not free images the pass is reading.
struct ScanImagesPin {
    ltr_ctx* ctx;
    explicit ScanImagesPin(ltr_ctx* c) : ctx(c) { ctx->scan_images_busy++; }
    ~ScanImagesPin() { ctx->scan_images_busy--; }
    ScanImagesPin(const ScanImagesPin&) = delete;
    ScanImagesPin& operator=(const ScanImagesPin&) = delete;
};

// The kept set with the scan images of a pass over [kf_begin, kf_end) -- found, completed or built, in launches over the whole range.
// The test image is the one of `coeff` (0: the constant threshold); the range image and the window table do not depend on it.
// A new set goes into an empty slot or the least recently used one, preferring a slot whose storage is already large enough; storage only
// grows.  *out = nullptr when the sets are off or the storage would exceed the budget: the pass then builds its images per launch.  The
// caller holds a ScanImagesPin.
static int scan_images_get(ltr_ctx* ctx, const PassPlan& p, const DevScanSet& scans, const DevPoses& poses, int kf_begin, int kf_end, bool need_pyr,
                           bool need_timg, bool pad, float coeff, ScanImageSet** out) {
    *out = nullptr;
    size_t budget = 0;
    if (!scan_image_cache_on(&budget)) return LTR_OK;
    const int K = kf_end - kf_begin;
    const int shortcut = p.fc.empty_scan_shortcut;
    const size_t npx = (size_t)p.npx;
    const size_t rimg_bytes = (size_t)K * npx * sizeof(uint32_t), pyr_bytes = rimg_bytes * kPyrLevels;
    const size_t timg_bytes = (size_t)K * (pad ? (size_t)p.fc.pad_npx : npx) * sizeof(uint32_t);
    // storage layout rimg | timg | pyr (256 B aligned): a set that needs the window table needs the whole block
    const size_t timg_off = (rimg_bytes + 255) / 256 * 256, pyr_off = timg_off + (timg_bytes + 255) / 256 * 256;
    const size_t need = need_pyr ? pyr_off + pyr_bytes : need_timg ? timg_off + timg_bytes : rimg_bytes;
    const ScanImageKey key{scans.serial, poses.serial, kf_begin, kf_end, p.g.rows, p.g.cols, ctx->cfg.transform_order, ctx->ext_identity ? 1 : 0,
                           ctx->cfg.fast_path, p.g.vfov, p.g.hfov};
    ScanImageSet* s = nullptr;
    for (ScanImageSet& c : ctx->scan_images)
        if (c.valid && c.key == key) s = &c;
    if (s && s->cap < need) scan_image_set_drop(*s);   // a part it lacks does not fit its storage: rebuild the set in a larger block
    if (!s || !s->valid) {
        if (!s) {   // empty before occupied, large enough before too small, then least recently used
            auto rank = [&](const ScanImageSet& c) { return std::make_tuple(c.valid ? 1 : 0, c.cap >= need ? 0 : 1, c.last_use); };
            s = &ctx->scan_images[0];
            for (ScanImageSet& c : ctx->scan_images) if (rank(c) < rank(*s)) s = &c;
        }
        scan_image_set_drop(*s);
        if (s->cap < need) {
            size_t others = 0;
            for (const ScanImageSet& c : ctx->scan_images) if (&c != s) others += c.cap;
            if (budget == 0) {
                size_t fr = 0, tot = 0;
                if (cudaMemGetInfo(&fr, &tot) != cudaSuccess) { cudaGetLastError(); return LTR_OK; }
                budget = (fr + ctx->cached_bytes + others + s->cap) / 4;
            }
            if (others + need > budget) return LTR_OK;
            dev_free(ctx, s->block);
            s->block = nullptr; s->cap = 0;
            const int rc = dev_alloc(ctx, &s->block, need);
            if (rc != LTR_OK) {   // out of memory within the budget (memory other processes took): build per launch
                if (rc != LTR_ERR_NOMEM) return rc;
                ctx->err.clear();
                return LTR_OK;
            }
            s->cap = need;
        }
        s->key = key;
    }
    char* base = (char*)s->block;
    const bool make_rimg = !s->valid;
    const bool make_pyr = need_pyr && s->pyr_shortcut != shortcut;
    uint32_t coeff_bits;
    std::memcpy(&coeff_bits, &coeff, sizeof(coeff_bits));
    const bool make_timg = need_timg && (s->timg_shortcut != shortcut || s->timg_coeff_bits != coeff_bits);
    s->rimg = (uint32_t*)base;
    s->timg = s->cap >= timg_off + timg_bytes ? (uint32_t*)(base + timg_off) : nullptr;
    s->pyr = s->cap >= pyr_off + pyr_bytes ? (float*)(base + pyr_off) : nullptr;
    if (make_rimg || make_pyr || make_timg) {
        s->valid = false;   // until the build is enqueued
        LTR_TRY(build_scan_images(ctx, p, scans, kf_begin, K, make_rimg, s->rimg, make_pyr ? s->pyr : nullptr, make_timg ? s->timg : nullptr, pad, coeff));
        s->valid = true;
        if (make_pyr) s->pyr_shortcut = shortcut;
        if (make_timg) { s->timg_shortcut = shortcut; s->timg_coeff_bits = coeff_bits; }
    }
    s->last_use = ++ctx->scan_images_tick;
    *out = s;
    return LTR_OK;
}

// Runs pass(allow_deferred, &overflowed) and, when the deferred true-minimum mode's candidate list filled up (8 M entries; never seen),
// repeats it in the immediate mode.
template <class Pass>
static int with_deferred_retry(Pass pass) {
    bool overflowed = false;
    LTR_TRY(pass(true, &overflowed));
    if (overflowed) LTR_TRY(pass(false, &overflowed));
    return LTR_OK;
}

}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_scan_images_release(ltr_ctx* ctx, int32_t free_storage) {
    ApiTrace tr__(ctx, "ltr_scan_images_release");
    if (!ctx) return LTR_ERR_INVALID;
    scan_images_release(ctx, 0, free_storage != 0);
    return LTR_OK;
}

// One run of remove_pass; allow_deferred: the true minimum may take the deferred mode.
static int remove_pass_impl(ltr_ctx* ctx, ltr_cloud map_h, ltr_scanset scans_h, ltr_poses poses_h, int32_t kf_begin, int32_t kf_end,
                            int32_t mode, float res_alpha, float thres, bool adaptive, float ball_radius, int32_t accumulate, int64_t* n_dynamic,
                            bool allow_deferred, bool* overflowed) {
    *overflowed = false;
    DevCloud* map;
    DevScanSet* scans;
    DevPoses* poses;
    LTR_TRY(cloud_get(ctx, map_h, &map));
    LTR_TRY(scanset_get(ctx, scans_h, &scans));
    LTR_TRY(poses_get(ctx, poses_h, &poses));
    if (mode != LTR_MODE_HD && mode != LTR_MODE_ND && mode != LTR_MODE_PD) return fail(ctx, LTR_ERR_INVALID, "unknown pass mode %d", mode);
    if (scans->K != poses->K) return fail(ctx, LTR_ERR_INVALID, "pose count %d != keyframe count %d (Session.cpp:117)", poses->K, scans->K);
    LTR_TRY(check_pass_range(ctx, *map, kf_begin, kf_end, scans->K));
    PassPlan p;
    LTR_TRY(plan_pass(ctx, res_alpha, kf_end - kf_begin, &p));
    LTR_TRY(cloud_ensure_flags(ctx, map));
    if (!accumulate && map->n > 0) LTR_CUDA(ctx, cudaMemsetAsync(map->flags, 0, (size_t)map->n, ctx->stream));
    const int64_t npx = p.npx;
    const int B = p.B;
    const bool cand = (mode != LTR_MODE_ND);
    const bool run = map->n > 0 && kf_end > kf_begin;
    int shortcut = 0;
    if (p.use_fast && cand && run) LTR_TRY(empty_scan_shortcut_ok(ctx, *map, *poses, kf_begin, kf_end, &shortcut));
    p.fc.empty_scan_shortcut = shortcut;
    const bool use_deferred = p.use_fast && !cand && allow_deferred;
    void* p_def = nullptr;
    ScratchGuard g_def(ctx, &p_def);
    DeferredArgs da{};
    if (use_deferred && run) LTR_TRY(deferred_alloc(ctx, B, npx, &p_def, &da));
    // tile culling (project_cull.cuh): scan-minus-map variants only, one keyframe per lane -> launches of at most 32 keyframes
    CullArgs ca{};
    // the sliding-window maxima cost 5 stores per pixel and keyframe: below one map point per pixel they cost more than the culling saves
    // (the small ND / PD candidate maps), so those passes project every pair
    const bool use_cull = p.use_fast && cand && ctx->cfg.fast_path >= 2 && B <= 32 && map->n >= kTilePts && map->n >= npx;
    void *p_tiles = nullptr, *p_pyr = nullptr;
    ScratchGuard g_tiles(ctx, &p_tiles), g_pyr(ctx, &p_pyr);
    // scan-minus-map with the short elevation path and a 360 degree field of view: the test image is guard-padded (FastCfg::pad_*) and always built;
    // so is the adaptive threshold's (scan_test_image_kernel)
    const bool pad = p.use_fast && cand && p.fc.pad_ok;
    const float timg_coeff = cand && adaptive ? thres : 0.0f;
    const bool need_timg = p.use_fast && cand && (shortcut || pad || adaptive);
    const int64_t timg_px = pad ? (int64_t)p.fc.pad_npx : npx;
    // the scan-side images come from a kept set built over the whole range (scan_images_get) or, without one, are built per launch
    ScanImagesPin pin(ctx);
    ScanImageSet* set = nullptr;
    if (run) LTR_TRY(scan_images_get(ctx, p, *scans, *poses, kf_begin, kf_end, use_cull, need_timg, pad, timg_coeff, &set));
    // the tile spheres bound culling's tiles and classify the fast path's ball tiles
    const bool use_ball = ball_radius != 0.0f && run;
    if (use_cull || (use_ball && p.use_fast)) LTR_TRY(tile_spheres(ctx, *map, &p_tiles));
    if (use_cull) {
        ca.enabled = 1;
        ca.tiles = (const float4*)p_tiles;
        ca.ntiles = tile_count(map->n);
        ca.pyr_stride = (unsigned)(kPyrLevels * npx);
        if (!set) LTR_TRY(dev_alloc(ctx, &p_pyr, (size_t)B * ca.pyr_stride * sizeof(float)));
    }
    BallLaunch bl;
    void* p_ball = nullptr;
    ScratchGuard g_ball(ctx, &p_ball);
    if (use_ball) LTR_TRY(ball_setup(ctx, p, *map, *poses, kf_begin, kf_end, ball_radius, (const float4*)p_tiles, &p_ball, &bl));
    LTR_TRY(pass_begin(ctx, p));
    if (run) {
        void *p_rimg = nullptr, *p_win = nullptr;
        ScratchGuard g_rimg(ctx, &p_rimg), g_win(ctx, &p_win);
        // per launch: the approximate running minimum (fast path), and without a kept set the scan image and the test image
        const int64_t per_kf = (p.use_fast ? npx : 0) + (set ? 0 : npx + (need_timg ? timg_px : 0));
        if (per_kf > 0) LTR_TRY(dev_alloc(ctx, &p_rimg, (size_t)B * per_kf * sizeof(uint32_t)));
        LTR_TRY(dev_alloc(ctx, &p_win, (size_t)B * npx * sizeof(uint64_t)));
        uint32_t* amin = p.use_fast ? (uint32_t*)p_rimg : nullptr;   // approximate running minimum (fast path only)
        uint32_t* l_rimg = set ? nullptr : (uint32_t*)p_rimg + (p.use_fast ? (size_t)B * npx : 0);
        uint32_t* l_timg = (set || !need_timg) ? nullptr : l_rimg + (size_t)B * npx;   // test image (padded, or pixels without a return can never flag)
        uint64_t* win = (uint64_t*)p_win;
        fill_u64_kernel<<<grid_for(B * npx, 256, ctx->sm_count * 8), 256, 0, ctx->stream>>>(win, cand ? kWinNone : kWinEmpty, B * npx);
        LTR_LAUNCH_CHECK(ctx);
        const Proj proj = cand ? Proj::kScanMinusMap : use_deferred ? Proj::kTrueMinDeferred : Proj::kTrueMin;
        for (int k0 = kf_begin; k0 < kf_end; k0 += B) {
            const int nb = std::min(B, kf_end - k0);
            const uint32_t *rimg, *test_img;
            if (set) {
                const size_t j = (size_t)(k0 - kf_begin);
                rimg = set->rimg + j * npx;
                test_img = need_timg ? set->timg + j * timg_px : rimg;
                if (use_cull) ca.pyr = set->pyr + j * ca.pyr_stride;
            } else {
                LTR_TRY(build_scan_images(ctx, p, *scans, k0, nb, true, l_rimg, use_cull ? (float*)p_pyr : nullptr, l_timg, pad, timg_coeff));
                rimg = l_rimg;
                test_img = need_timg ? l_timg : l_rimg;
                if (use_cull) ca.pyr = (const float*)p_pyr;
            }
            if (use_ball) bl.args.centre = (const float4*)p_ball + (k0 - kf_begin);
            LTR_TRY(project_map(ctx, p, *map, *poses, k0, nb, proj, rimg, test_img, thres, adaptive, win, amin, ca, da, bl));
            const unsigned rb = (unsigned)((nb * npx + 255) / 256);
            const auto resolve = with_bools([](auto c, auto ad) { return resolve_kernel<c, ad>; }, cand, adaptive);
            resolve<<<rb, 256, 0, ctx->stream>>>(rimg, win, nb * npx, thres, map->flags);
            LTR_LAUNCH_CHECK(ctx);
        }
    }
    g_tiles.release();
    g_pyr.release();
    g_ball.release();
    LTR_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    if (n_dynamic) LTR_TRY(count_flags(ctx, map->flags, map->n, n_dynamic));
    unsigned int h_over = 0;
    if (da.overflow) LTR_CUDA(ctx, cudaMemcpyAsync(&h_over, da.overflow, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
    if (da.overflow) { LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); *overflowed = h_over != 0; }
    g_def.release();
    pass_end(ctx, p, 0, 12.0 * (double)map->n + (double)map->n / 8.0, map->n, kf_end - kf_begin);
    return LTR_OK;
}

// The remove pass of the three entry points.  adaptive: `thres` is the coefficient c of the pixel threshold fl(c s), else the constant
// threshold.  ball_radius > 0: keyframe k sees only the map points within that radius of its pose's f32 translation (ball_setup); 0: the
// full map.  ND (true per-pixel minimum) runs in the deferred mode of project_fast.cuh unless the flags accumulate into earlier ones (a run
// whose overflow list filled up would have to be undone).
static int remove_pass(ltr_ctx* ctx, ltr_cloud map_h, ltr_scanset scans_h, ltr_poses poses_h, int32_t kf_begin, int32_t kf_end, int32_t mode,
                       float res_alpha, float thres, bool adaptive, float ball_radius, int32_t accumulate, int64_t* n_dynamic) {
    // NaN fails both comparisons
    if (adaptive && !(thres > 0.0f && thres < 1.0f)) return fail(ctx, LTR_ERR_INVALID, "adaptive coefficient %g outside (0, 1)", (double)thres);
    return with_deferred_retry([&](bool allow_deferred, bool* overflowed) {
        return remove_pass_impl(ctx, map_h, scans_h, poses_h, kf_begin, kf_end, mode, res_alpha, thres, adaptive, ball_radius, accumulate, n_dynamic,
                                allow_deferred && !accumulate, overflowed);
    });
}

int ltr_remove_pass(ltr_ctx* ctx, ltr_cloud map_h, ltr_scanset scans_h, ltr_poses poses_h, int32_t kf_begin, int32_t kf_end,
                    int32_t mode, float res_alpha, float diff_thres, int32_t accumulate, int64_t* n_dynamic) {
    ApiTrace tr__(ctx, "ltr_remove_pass");
    if (!ctx) return LTR_ERR_INVALID;
    return remove_pass(ctx, map_h, scans_h, poses_h, kf_begin, kf_end, mode, res_alpha, diff_thres, false, 0.0f, accumulate, n_dynamic);
}

int ltr_remove_pass_adaptive(ltr_ctx* ctx, ltr_cloud map_h, ltr_scanset scans_h, ltr_poses poses_h, int32_t kf_begin, int32_t kf_end,
                             int32_t mode, float res_alpha, float adaptive_coeff, int32_t accumulate, int64_t* n_dynamic) {
    ApiTrace tr__(ctx, "ltr_remove_pass_adaptive");
    if (!ctx) return LTR_ERR_INVALID;
    return remove_pass(ctx, map_h, scans_h, poses_h, kf_begin, kf_end, mode, res_alpha, adaptive_coeff, true, 0.0f, accumulate, n_dynamic);
}

int ltr_remove_pass_ball(ltr_ctx* ctx, ltr_cloud map_h, ltr_scanset scans_h, ltr_poses poses_h, int32_t kf_begin, int32_t kf_end,
                         int32_t mode, float res_alpha, float diff_thres, float adaptive_coeff, float ball_radius, int32_t accumulate, int64_t* n_dynamic) {
    ApiTrace tr__(ctx, "ltr_remove_pass_ball");
    if (!ctx) return LTR_ERR_INVALID;
    // NaN fails every comparison
    if (!(ball_radius > 0.0f && ball_radius <= 3.4028235e38f)) return fail(ctx, LTR_ERR_INVALID, "ball radius %g is not finite and > 0", (double)ball_radius);
    const bool adaptive = adaptive_coeff != 0.0f;   // else the constant threshold diff_thres
    return remove_pass(ctx, map_h, scans_h, poses_h, kf_begin, kf_end, mode, res_alpha, adaptive ? adaptive_coeff : diff_thres, adaptive, ball_radius,
                       accumulate, n_dynamic);
}

// An overflowed run (*overflowed) frees its output again and leaves *out unwritten.
static int parse_projected_impl(ltr_ctx* ctx, ltr_cloud map_h, ltr_poses poses_h, int32_t kf_begin, int32_t kf_end, float res_alpha, ltr_scanset* out,
                                bool allow_deferred, bool* overflowed) {
    *overflowed = false;
    DevCloud* map;
    DevPoses* poses;
    LTR_TRY(cloud_get(ctx, map_h, &map));
    LTR_TRY(poses_get(ctx, poses_h, &poses));
    LTR_TRY(check_pass_range(ctx, *map, kf_begin, kf_end, poses->K));
    const int K = kf_end - kf_begin;
    PassPlan p;
    LTR_TRY(plan_pass(ctx, res_alpha, K, &p));
    const int64_t npx = p.npx;
    const DevCloud mapc = *map;
    const DevPoses posc = *poses;
    std::vector<int64_t> off((size_t)K + 1, 0);
    LTR_TRY(pass_begin(ctx, p));
    void *p_list = nullptr, *p_cnt = nullptr, *p_def = nullptr;
    ScratchGuard g_list(ctx, &p_list), g_cnt(ctx, &p_cnt), g_def(ctx, &p_def);
    DeferredArgs da{};
    const bool use_deferred = p.use_fast && allow_deferred;
    if (K > 0 && mapc.n > 0) {
        const int B = p.B;
        if (use_deferred) LTR_TRY(deferred_alloc(ctx, B, npx, &p_def, &da));
        void *p_win = nullptr, *p_amin = nullptr, *p_tiles = nullptr, *p_keys = nullptr;
        ScratchGuard g_win(ctx, &p_win), g_amin(ctx, &p_amin), g_tiles(ctx, &p_tiles), g_keys(ctx, &p_keys);
        LTR_TRY(dev_alloc(ctx, &p_win, (size_t)B * npx * sizeof(uint64_t)));
        if (p.use_fast && !use_deferred) LTR_TRY(dev_alloc(ctx, &p_amin, (size_t)B * npx * sizeof(uint32_t)));   // the deferred mode keeps `best` instead
        uint32_t* amin = (uint32_t*)p_amin;
        // deferred mode: the tiles are claimed near to far from each launch's keyframes (DeferredArgs::order); their bounding spheres
        // are computed once per call
        const bool use_order = use_deferred && mapc.n >= kTilePts;
        const long long ntiles = tile_count(mapc.n);
        uint64_t* keys = nullptr;
        if (use_order) {
            LTR_TRY(tile_spheres(ctx, mapc, &p_tiles));
            LTR_TRY(dev_alloc(ctx, &p_keys, (size_t)ntiles * 2 * sizeof(uint64_t)));
            keys = (uint64_t*)p_keys;
        }
        const CullArgs no_cull{};
        LTR_TRY(dev_alloc(ctx, &p_list, (size_t)K * npx * sizeof(uint32_t)));
        const int nchunk = (int)((npx + kParseChunk - 1) / kParseChunk);
        LTR_TRY(dev_alloc(ctx, &p_cnt, ((size_t)K + (size_t)B * nchunk) * sizeof(unsigned int)));
        unsigned int* chunk_cnt = (unsigned int*)p_cnt + K;
        uint64_t* win = (uint64_t*)p_win;
        fill_u64_kernel<<<grid_for(B * npx, 256, ctx->sm_count * 8), 256, 0, ctx->stream>>>(win, kWinEmpty, B * npx);
        LTR_LAUNCH_CHECK(ctx);
        for (int k0 = 0; k0 < K; k0 += B) {
            const int nb = std::min(B, K - k0);
            if (use_order) {
                // reference origin of the launch: the mean sensor origin of its keyframes (KfFast::chi)
                double o[3] = {0.0, 0.0, 0.0};
                for (int k = 0; k < nb; ++k)
                    for (int d = 0; d < 3; ++d) o[d] += (double)posc.h_fast[(size_t)(kf_begin + k0 + k) * 16 + 9 + d] / nb;
                tile_order_key_kernel<<<(unsigned)((ntiles + 255) / 256), 256, 0, ctx->stream>>>((const float4*)p_tiles, ntiles, (float)o[0], (float)o[1],
                                                                                                  (float)o[2], keys);
                LTR_LAUNCH_CHECK(ctx);
                uint64_t* sorted = nullptr;
                LTR_TRY(radix_sort_pairs(ctx, keys, keys + ntiles, nullptr, nullptr, ntiles, 32, 48, &sorted, nullptr));
                da.order = (const unsigned long long*)sorted;
            }
            LTR_TRY(project_map(ctx, p, mapc, posc, kf_begin + k0, nb, use_deferred ? Proj::kTrueMinDeferred : Proj::kTrueMin, nullptr, nullptr, 0.0f,
                                false, win, amin, no_cull, da));
            parse_count_kernel<<<dim3((unsigned)nchunk, (unsigned)nb), 1024, 0, ctx->stream>>>(win, (int)npx, nchunk, chunk_cnt);
            LTR_LAUNCH_CHECK(ctx);
            parse_compact_kernel<<<dim3((unsigned)nchunk, (unsigned)nb), 1024, 0, ctx->stream>>>(win, (int)npx, nchunk, chunk_cnt, (uint32_t*)p_list + (size_t)k0 * npx,
                                                                                              (unsigned int*)p_cnt + k0);
            LTR_LAUNCH_CHECK(ctx);
        }
        g_win.release();
        g_amin.release();
        g_tiles.release();
        g_keys.release();
        std::vector<unsigned int> cnt((size_t)K);
        unsigned int h_over = 0;
        LTR_CUDA(ctx, cudaMemcpyAsync(cnt.data(), p_cnt, (size_t)K * sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
        if (da.overflow) LTR_CUDA(ctx, cudaMemcpyAsync(&h_over, da.overflow, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        g_def.release();
        if (h_over) *overflowed = true;
        for (int k = 0; k < K; ++k) off[k + 1] = off[k] + cnt[k];
    }
    ScanSetOwner o;
    LTR_TRY(scanset_new(ctx, off, &o));
    DevScanSet& os = ctx->scansets[o.get()];
    if (os.pts.n > 0) {
        parse_emit_kernel<<<(unsigned)((os.pts.n + 255) / 256), 256, 0, ctx->stream>>>(view(mapc), posc.d, kf_begin, os.d_off, K, (const uint32_t*)p_list,
            (int)npx, ctx->d_ext, ctx->ext_identity ? 1 : 0, ctx->cfg.transform_order, os.pts);
        LTR_LAUNCH_CHECK(ctx);
    }
    g_list.release();
    g_cnt.release();
    LTR_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
    LTR_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
    pass_end(ctx, p, 4, 12.0 * (double)mapc.n, mapc.n, K);
    if (!*overflowed) *out = o.release();
    return LTR_OK;
}

int ltr_parse_projected(ltr_ctx* ctx, ltr_cloud map_h, ltr_poses poses_h, int32_t kf_begin, int32_t kf_end, float res_alpha, ltr_scanset* out) {
    ApiTrace tr__(ctx, "ltr_parse_projected");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    return with_deferred_retry([&](bool allow_deferred, bool* overflowed) {
        return parse_projected_impl(ctx, map_h, poses_h, kf_begin, kf_end, res_alpha, out, allow_deferred, overflowed);
    });
}

int ltr_debug_pixel_index(ltr_ctx* ctx, const float* xyz, int64_t n, int32_t rows, int32_t cols, int32_t* row, int32_t* col, float* range,
                          float* az, float* el) {
    ApiTrace tr__(ctx, "ltr_debug_pixel_index");
    if (!ctx || !xyz || n < 0) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    if (n == 0) return LTR_OK;
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    const size_t bytes = (size_t)n * (3 + 5) * 4;
    LTR_TRY(dev_alloc(ctx, &p, bytes));
    float* d_xyz = (float*)p;
    int* d_row = (int*)(d_xyz + 3 * n);
    int* d_col = d_row + n;
    float* d_rng = (float*)(d_col + n);
    float* d_az = d_rng + n;
    float* d_el = d_az + n;
    LTR_CUDA(ctx, cudaMemcpyAsync(d_xyz, xyz, (size_t)n * 12, cudaMemcpyHostToDevice, ctx->stream));
    const ImgShape g{rows, cols, ctx->cfg.vfov_deg, ctx->cfg.hfov_deg};
    debug_pixel_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_xyz, n, g, d_row, d_col, d_rng, d_az, d_el);
    LTR_LAUNCH_CHECK(ctx);
    if (row) LTR_CUDA(ctx, cudaMemcpyAsync(row, d_row, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (col) LTR_CUDA(ctx, cudaMemcpyAsync(col, d_col, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (range) LTR_CUDA(ctx, cudaMemcpyAsync(range, d_rng, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (az) LTR_CUDA(ctx, cudaMemcpyAsync(az, d_az, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (el) LTR_CUDA(ctx, cudaMemcpyAsync(el, d_el, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}

int ltr_debug_margins(ltr_ctx* ctx, float res_alpha, float* m) {
    if (!ctx || !m) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    PassPlan plan;
    LTR_TRY(plan_pass(ctx, res_alpha, 1, &plan));
    const FastCfg& fc = plan.fc;
    m[0] = fc.m_col_a; m[1] = fc.m_col_b; m[2] = fc.m_row; m[3] = fc.m_r_rel; m[4] = fc.m_r_abs; m[5] = (float)fc.el_direct;
    m[6] = (float)((fc.m_col_a + fc.m_col_b) / kMarginSafety); m[7] = (float)(fc.m_row / kMarginSafety);
    m[8] = fc.az_seam_lim;
    return LTR_OK;
}

int ltr_debug_atan_sweep(ltr_ctx* ctx, int32_t which, double* max_abs_err, float* arg_at_max) {
    ApiTrace tr__(ctx, "ltr_debug_atan_sweep");
    if (!ctx || !max_abs_err || (which != 0 && which != 1)) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, 16));
    LTR_CUDA(ctx, cudaMemsetAsync(p, 0, 16, ctx->stream));
    const uint32_t last = which == 0 ? 0x3F800000u : 0x3F000000u;   // 1.0f / 0.5f
    atan_sweep_kernel<<<ctx->sm_count * 16, 256, 0, ctx->stream>>>(which, last, (unsigned long long*)p, (uint32_t*)((char*)p + 8));
    LTR_LAUNCH_CHECK(ctx);
    unsigned long long h[2] = {0, 0};
    LTR_CUDA(ctx, cudaMemcpyAsync(h, p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::memcpy(max_abs_err, &h[0], 8);
    if (arg_at_max) { const uint32_t b = (uint32_t)h[1]; std::memcpy(arg_at_max, &b, 4); }
    return LTR_OK;
}

int ltr_debug_scan_rimg(ltr_ctx* ctx, ltr_scanset scans_h, int32_t kf, float res_alpha, float* out) {
    ApiTrace tr__(ctx, "ltr_debug_scan_rimg");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevScanSet* scans;
    LTR_TRY(scanset_get(ctx, scans_h, &scans));
    if (kf < 0 || kf >= scans->K) return fail(ctx, LTR_ERR_INVALID, "keyframe %d outside [0,%d)", kf, scans->K);
    PassPlan plan;
    LTR_TRY(plan_pass(ctx, res_alpha, 1, &plan));
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, (size_t)plan.npx * sizeof(uint32_t)));
    LTR_TRY(scan_rimg(ctx, plan, *scans, kf, 1, (uint32_t*)p));
    LTR_CUDA(ctx, cudaMemcpyAsync(out, p, (size_t)plan.npx * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}

int ltr_debug_fast_project(ltr_ctx* ctx, const float* xyz, int64_t n, const double* inv_pose16, float res_alpha, float* out8, float* margins4) {
    ApiTrace tr__(ctx, "ltr_debug_fast_project");
    if (!ctx || !xyz || !inv_pose16 || !out8 || n < 0) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    PassPlan plan;
    LTR_TRY(plan_pass(ctx, res_alpha, 1, &plan));
    const FastCfg& fc = plan.fc;
    if (margins4) { margins4[0] = fc.m_col_a; margins4[1] = fc.m_col_b; margins4[2] = fc.m_row; margins4[3] = fc.m_r_rel; }
    if (n == 0) return LTR_OK;
    ltr_poses ph;
    double id[16];
    for (int i = 0; i < 16; ++i) id[i] = (i % 5 == 0) ? 1.0 : 0.0;
    LTR_TRY(ltr_poses_upload(ctx, id, inv_pose16, 1, &ph));
    PosesOwner g_ph(ctx, ph);
    const DevPoses pp = ctx->poses[ph];
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, (size_t)n * (3 + 8) * sizeof(float)));
    float* d_xyz = (float*)p;
    float* d_out = d_xyz + 3 * n;
    LTR_CUDA(ctx, cudaMemcpyAsync(d_xyz, xyz, (size_t)n * 12, cudaMemcpyHostToDevice, ctx->stream));
    const auto kern = with_bools([](auto el) { return debug_fast_kernel<el>; }, fc.el_direct != 0);
    kern<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_xyz, n, pp.d_fast, pp.d, ctx->d_ext, ctx->ext_identity ? 1 : 0, ctx->cfg.transform_order,
                                                               plan.g, fc, d_out);
    LTR_LAUNCH_CHECK(ctx);
    LTR_CUDA(ctx, cudaMemcpyAsync(out8, d_out, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}

}  // extern "C"
