// Exactness-preserving fast rejection path of the map projection (used by ltr_remove_pass / ltr_parse_projected).
//
// The reference arithmetic per (map point, keyframe) -- two double-precision transforms with float rounding,
// fdlibm atan2f twice, IEEE divisions and square roots, double rad2deg (ltremovert/src/utility.cpp:38-56, 64-72,
// 118-123) -- costs ~500 non-FMA instructions.  Almost every (point, keyframe) pair has NO effect on the result:
//   * scan-minus-map variants (HD / revert / PD): only points with scan_range - range > thres can win the per-pixel
//     atomic (SURVEY.md A.2); static structure (range ~ scan range) and occluded points never do;
//   * true-min variants (ND, visible-point extraction): only points at most as near as the pixel's current minimum.
// So each pair is first evaluated with ~90 FMA-based float instructions whose error against the reference value is
// bounded (margins below).  The pair is DROPPED only if, for every value inside the error bound, the reference
// arithmetic would also have produced "no effect"; otherwise it is queued (warp-aggregated, shared memory) and the
// queue is drained 32 entries at a time through the bit-exact path of ref_math.cuh.  Results are therefore identical
// to the all-exact kernel; tests/test_gpu_fastpath.py checks the margins against measured deviations and
// the flags / visible points against the oracle with the fast path on and off.
#pragma once
#include "ref_math.cuh"

namespace ltr {

// Per-keyframe single-precision constants: q ~= A * (p - c_hi) - A * c_lo, c = c_hi + c_lo = sensor origin in the map frame.
// Subtracting the origin first makes the rounding error proportional to the RANGE, not to the map coordinates.
struct KfFast { float A[9]; float chi[3]; float tlo[3]; float ok; };  // 16 floats: q ~= A (p - c_hi) - t_lo; ok == 0 -> exact path only

struct FastCfg {
    float col_scale, col_off;   // V_col ~= az * col_scale + col_off   (= C * ((deg(az) + H/2) / H))
    float row_scale, row_off;   // V_row ~= row_off - el * row_scale   (= R * (1 - (deg(el) + V/2) / V))
    float m_col_a, m_col_b;     // column margin [px] = m_col_a + m_col_b * (r / rho)
    float m_row;                // row margin [px]
    float m_r_rel, m_r_abs;     // range margin [m] = m_r_abs + m_r_rel * r
    int empty_scan_shortcut;    // 1: no map point can be >= 9000 m from a keyframe -> pixels without a scan return never flag
    // folded forms of the above, so that the hot loop takes them straight from the constant bank
    float lim_c, lim_r;         // 0.5 - m_col_a, 0.5 - m_row
    float rel_m1;               // m_r_rel - 1
    float mr2_rel, mr2_abs;     // 2 * m_r_rel, 2 * m_r_abs
    float neg_row_scale;
    int el_direct;              // 1: |elevation| beyond atan(0.5) clamps to the first / last row with room to spare -> short elevation path
    // guard-padded test image of the scan-minus-map variant with the short elevation path (scan_test_image_kernel): pad_g rows above and
    // below replicate the first / last row, and one guard column follows the last; pixel (r, c) is at (r + pad_g) * (cols + 1) + c
    int pad_ok;                 // 1: el_direct and a 360 degree field of view (columns in [0, cols], the seam at columns 0 / cols)
    int pad_g;                  // rows the short path can reach beyond either edge of the image
    int pad_npx;                // (rows + 2 pad_g) * (cols + 1): padded pixels per keyframe
    uint32_t pad_w;             // cols + 1
    uint32_t pad_bias;          // 0x4B400000 (cols + 2) - pad_g (cols + 1), modulo 2^32 (see map_project_fast_kernel)
    uint32_t pad_last;          // pad_npx - 1
    float az_seam_lim;          // pi - 0.5 / col_scale: a fast azimuth at least this close to +-pi is never certain (map_project_fast_kernel)
};

// ---------------------------------------------------------------------------------------------------------------------------
// Error budget of the fast evaluation against the REFERENCE's own pre-round pixel coordinates and range (DESIGN.md section 4.1
// derives each line; u = 2^-24 is the unit roundoff of a correctly rounded f32 operation, MUFU.RCP is within 2^-23 and MUFU.RSQ
// within 2^-22.4 relative (PTX ISA, rcp/rsqrt.approx.ftz.f32); tests/test_gpu_fastpath.py sweeps EVERY float of [0, 1] through both
// polynomials and asserts the two constants marked (*), and checks measured deviations of whole projections against the margins).
//   q_fast:  dx = fl(p - c_hi) (u |d|), three chained FMAs with f32-rounded matrix entries  ->  |dq_i| <= 5 u r per component
//   q_ref :  double transform rounded once to f32                                               ->  |dq_i| <= u |q_i|
// Azimuth [rad]                                            fast                                  reference chain (utility.cpp:46, 53-56, 123)
//   from dq                                                5 sqrt(2) u r / rho = 4.3e-7 r/rho    u                      = 0.6e-7
//   a = min * rcp(max): (2^-23 + u) * a / (1 + a^2)        0.9e-7                                atan2f (fdlibm, < 1 ulp of pi) 2.4e-7
//   7-coefficient polynomial incl. its f32 evaluation (*)  6.8e-7                                rad2deg: f64, rounded to f32   1.9e-7
//   quadrant fix-ups (f32 constants and subtractions)      3.2e-7                                deg + H/2 (0.5 ulp of 360)     2.7e-7
//   sum                                                    1.09e-6 + 4.3e-7 r/rho                7.6e-7
//   pixel-space roundings (fma / divide / scale)           1.5 u C                               2 u C
// Elevation [rad], short path |qz / rho| <= 0.5
//   from dq                                                5.2e-7                                u                      = 0.6e-7
//   t = qz * rsq(rho^2): (2^-22.4 + u) * t / (1 + t^2)     1.0e-7                                atan2f (< 1 ulp of pi/2)       1.2e-7
//   5-coefficient polynomial incl. its f32 evaluation (*)  0.9e-7                                rad2deg + (deg + V/2)          1.6e-7
//   sum                                                    7.1e-7                                3.4e-7
//   pixel-space roundings                                  1.5 u R                               3 u R
// Range (relative): MUFU.RSQ 1.8e-7 + r^2 accumulation 3 u + dq 5 sqrt(3) u = 9.4e-7 (fast) + 2.5 u (reference) = 1.1e-6
// The margins below are these sums times kMarginSafety.  NaN or infinity anywhere fails every comparison -> exact path.
// ---------------------------------------------------------------------------------------------------------------------------
constexpr double kMarginSafety = 1.5;
constexpr double kU = 5.9604644775390625e-08;
constexpr double kAzPolyErr = 6.8e-7;    // (*) max |fast_atan01(a) - atan(a)| over all floats a in [0, 1]
constexpr double kElPolyErr = 0.9e-7;    // (*) max |fast_atan_half(t) - atan(t)| over all floats |t| <= 0.5
constexpr double kAzFixed = (kU + 2.4e-7 + 1.9e-7 + 2.7e-7) + (0.9e-7 + kAzPolyErr + 3.2e-7);   // rad, independent of r/rho
constexpr double kAzPerRhoInvR = 4.3e-7;                                                        // rad per unit of r/rho
constexpr double kElFixed = (kU + 1.2e-7 + 1.6e-7) + (5.2e-7 + 1.0e-7 + kElPolyErr);            // rad
constexpr double kElFixedGeneral = (kU + 1.2e-7 + 1.6e-7) + (5.2e-7 + 1.2e-7 + 0.9e-7 + kAzPolyErr + 1.0e-7);   // general path: rho = rho^2 * rsq, min * rcp(max), azimuth polynomial, pi/2 fix-up
constexpr double kRangeRel = 1.1e-6;

__host__ inline FastCfg make_fast_cfg(int rows, int cols, float vfov, float hfov, int empty_scan_shortcut) {
    FastCfg f;
    const double kPi = 3.14159265358979323846;
    const double ppr_c = (double)cols * 180.0 / (kPi * (double)hfov);   // pixels per radian
    const double ppr_r = (double)rows * 180.0 / (kPi * (double)vfov);
    f.col_scale = (float)ppr_c; f.col_off = 0.5f * (float)cols;
    f.row_scale = (float)ppr_r; f.row_off = 0.5f * (float)rows;
    // short elevation path: an elevation of +-atan(0.5) must land at least one full pixel outside the image, so that clamping t = qz / rho
    // to +-0.5 cannot move a point across a row boundary
    const double half_v = 0.5 * (double)vfov * kPi / 180.0;
    f.el_direct = (std::atan(0.5) - half_v) * ppr_r >= 1.0 ? 1 : 0;
    f.m_col_a = (float)(kMarginSafety * (ppr_c * kAzFixed + (double)cols * 3.5 * kU));
    f.m_col_b = (float)(kMarginSafety * ppr_c * kAzPerRhoInvR);
    f.m_row = (float)(kMarginSafety * (ppr_r * (f.el_direct ? kElFixed : kElFixedGeneral) + (double)rows * 4.5 * kU));
    f.m_r_rel = (float)(kMarginSafety * kRangeRel); f.m_r_abs = 5.0e-6f;
    f.empty_scan_shortcut = empty_scan_shortcut;
    f.lim_c = 0.5f - f.m_col_a; f.lim_r = 0.5f - f.m_row;
    f.rel_m1 = f.m_r_rel - 1.0f;
    f.mr2_rel = 2.0f * f.m_r_rel; f.mr2_abs = 2.0f * f.m_r_abs;
    f.neg_row_scale = -f.row_scale;
    // half a pixel of azimuth short of the seam (rounding the double to f32 moves it by at most 1.2e-7 rad, a thousandth of a pixel
    // at 1 000 px per radian; the band only has to hold the pairs within their column margin of the seam, see the kernel)
    f.az_seam_lim = (float)(kPi - 0.5 / ppr_c);
    // the short path's elevation is |fast_atan_half(t)| <= atan(0.5) + kElPolyErr; the rows it rounds to, with 1e-3 px for the f32 pixel arithmetic
    const double el_max = std::atan(0.5) + kElPolyErr;
    const int r_top = (int)std::floor(0.5 * rows - el_max * ppr_r - 1.0e-3 + 0.5);
    const int r_bot = (int)std::floor(0.5 * rows + el_max * ppr_r + 1.0e-3 + 0.5);
    f.pad_ok = (f.el_direct && hfov == 360.0f) ? 1 : 0;
    f.pad_g = f.pad_ok ? std::max(std::max(-r_top, r_bot - (rows - 1)), 0) : 0;
    f.pad_npx = (rows + 2 * f.pad_g) * (cols + 1);
    f.pad_w = (uint32_t)(cols + 1);
    f.pad_bias = 0x4B400000u * (uint32_t)(cols + 2) - (uint32_t)(f.pad_g * (cols + 1));   // bits of 1.5 * 2^23 + i are 0x4B400000 + i for |i| < 2^22
    f.pad_last = (uint32_t)f.pad_npx - 1u;
    return f;
}

// single-instruction approximations (MUFU) without the denormal fix-up sequences of rsqrtf()/__fdividef()
LTR_DEV float mufu_rsq(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
LTR_DEV float mufu_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// atan(a) for a in [0, 1]: a * P(a^2), 7 coefficients (near-minimax fit of atan(sqrt(z)) / sqrt(z) on [0, 1]); the error constant
// kAzPolyErr is asserted over every float of [0, 1] by tests/test_gpu_fastpath.py::test_atan_polynomials_exhaustive
LTR_DEV float fast_atan01(float a) {
    const float z = __fmul_rn(a, a);
    float p = 0.008006718009710312f;
    p = __fmaf_rn(p, z, -0.037442438304424286f);
    p = __fmaf_rn(p, z, 0.0843534842133522f);
    p = __fmaf_rn(p, z, -0.1351214498281479f);
    p = __fmaf_rn(p, z, 0.1988731473684311f);
    p = __fmaf_rn(p, z, -0.3332701325416565f);
    p = __fmaf_rn(p, z, 0.9999994039535522f);
    return __fmul_rn(p, a);
}

// atan(t) for |t| <= 0.5: t * P(t^2), 5 coefficients (fit on z in [0, 0.25]); odd in t, so the sign comes for free
LTR_DEV float fast_atan_half(float t) {
    const float z = __fmul_rn(t, t);
    float p = 0.06964161992073059f;
    p = __fmaf_rn(p, z, -0.13479125499725342f);
    p = __fmaf_rn(p, z, 0.199324369430542f);
    p = __fmaf_rn(p, z, -0.33331313729286194f);
    p = __fmaf_rn(p, z, 0.9999998807907104f);
    return __fmul_rn(p, t);
}

struct FastProj { float az, el, r, rho_inv_r; };  // rho_inv_r = r / rho

// approximate cart2sph of a point in the sensor frame.  kElDirect: elevation from t = qz / rho clamped to +-0.5 (FastCfg::el_direct).
template <bool kElDirect = false>
LTR_DEV FastProj fast_sph(float qx, float qy, float qz) {
    const float rho2 = __fmaf_rn(qy, qy, __fmul_rn(qx, qx));
    const float r2 = __fmaf_rn(qz, qz, rho2);
    const float irho = mufu_rsq(rho2), ir = mufu_rsq(r2);
    FastProj o;
    o.r = __fmul_rn(r2, ir);
    o.rho_inv_r = __fmul_rn(o.r, irho);
    // azimuth = atan2(qy, qx); 0/0 -> NaN (NaN always routes to the exact path)
    {
        const float ax = fabsf(qx), ay = fabsf(qy);
        float t = fast_atan01(__fmul_rn(fminf(ax, ay), mufu_rcp(fmaxf(ax, ay))));
        if (ay > ax) t = __fsub_rn(1.57079632679f, t);
        if (qx < 0.0f) t = __fsub_rn(3.14159265359f, t);
        o.az = copysignf(t, qy);
    }
    // elevation = atan2(qz, rho), rho >= 0
    if (kElDirect) {
        // beyond +-atan(0.5) the row index is clamped anyway (make_fast_cfg checked the room); fminf / fmaxf drop a NaN of qz * irho
        // (rho == 0), but then the azimuth above is NaN as well and the pair goes to the exact path
        const float t = fminf(fmaxf(__fmul_rn(qz, irho), -0.5f), 0.5f);
        o.el = fast_atan_half(t);
    } else {
        const float rho = __fmul_rn(rho2, irho);
        const float az_ = fabsf(qz);
        float t = fast_atan01(__fmul_rn(fminf(rho, az_), mufu_rcp(fmaxf(rho, az_))));
        if (az_ > rho) t = __fsub_rn(1.57079632679f, t);
        o.el = copysignf(t, qz);
    }
    return o;
}

// kf: A[0..8], c_hi[9..11], t_lo[12..14] = A * c_lo, ok[15]:  q ~= A * (p - c_hi) - t_lo
template <bool kElDirect = false>
LTR_DEV FastProj fast_project(const float* __restrict__ kf, float x, float y, float z) {
    const float dx = __fsub_rn(x, kf[9]), dy = __fsub_rn(y, kf[10]), dz = __fsub_rn(z, kf[11]);
    const float qx = __fmaf_rn(kf[2], dz, __fmaf_rn(kf[1], dy, __fmaf_rn(kf[0], dx, -kf[12])));
    const float qy = __fmaf_rn(kf[5], dz, __fmaf_rn(kf[4], dy, __fmaf_rn(kf[3], dx, -kf[13])));
    const float qz = __fmaf_rn(kf[8], dz, __fmaf_rn(kf[7], dy, __fmaf_rn(kf[6], dx, -kf[14])));
    return fast_sph<kElDirect>(qx, qy, qz);
}

// Rounds a pre-round pixel coordinate when that is certain: returns true and the clamped index iff every value within
// +-margin of v rounds (half away from zero) to the same integer.  NaN -> false.  |v| < 2^22 (pixel coordinates).
LTR_DEV bool certain_round(float v, float margin, int hi, int* idx) {
    const float kMagic = 12582912.0f;                         // 1.5 * 2^23: v + kMagic has the nearest integer in its low mantissa bits
    const float y = __fadd_rn(v, kMagic);
    const float n = __fsub_rn(y, kMagic);                     // nearest integer (ties to even; ties are inside the margin anyway)
    const float d = fabsf(__fsub_rn(v, n));                   // distance to the nearest integer, in [0, 0.5]
    *idx = min(max(__float_as_int(y) - 0x4B400000, 0), hi);
    return d < __fsub_rn(0.5f, margin);                       // i.e. farther than `margin` from the rounding boundary n +- 0.5
}

constexpr uint32_t kNoPointBitsF = 0x461C4000u;  // 10000.0f

// queue entry: [63:32] map index | [31:14] pixel (row * cols + col, < 2^18) | [13:0] keyframe within the batch
LTR_DEV uint64_t q_pack(uint32_t i, uint32_t px, uint32_t k) { return ((uint64_t)i << 32) | (px << 14) | k; }

// The discrepancy threshold of a pixel whose scan range is s (calcDescrepancyAndParseDynamicPointIdx, Removerter.cpp:393-398): the constant
// `thres`, or with kAdaptive the range-proportional fl(c s) of the reference's commented-out line 396, the coefficient c passed in `thres`.
template <bool kAdaptive>
LTR_DEV float pixel_thres(float thres, float s) { return kAdaptive ? fm(thres, s) : thres; }

// Offers the exact key (range r, map index i) to pixel px of the winner image.  kCandidatesOnly: only a candidate (scan - r > t, t the
// pixel's threshold, pixel_thres) enters, and with the empty-scan shortcut a pixel without a scan return turns every pair away (diff > 200
// for every map point there, whatever t is).  A key that is not below the pixel's current one skips the atomic.
template <bool kCandidatesOnly, bool kAdaptive = false>
LTR_DEV void offer(uint64_t* __restrict__ win, size_t px, float r, uint32_t i, const uint32_t* __restrict__ scan_rimg, float thres, int shortcut,
                   unsigned* n_atomics) {
    const uint64_t packed = ((uint64_t)__float_as_uint(r) << 32) | i;
    if (kCandidatesOnly) {
        const uint32_t sb = scan_rimg[px];
        if (shortcut && sb == kNoPointBitsF && r < 9000.0f) return;
        const float s = __uint_as_float(sb);
        if (!(fs(s, r) > pixel_thres<kAdaptive>(thres, s))) return;
    }
    if (packed < win[px]) { atomicMin((unsigned long long*)&win[px], (unsigned long long)packed); ++*n_atomics; }
}

// The reference arithmetic of one pair: map point i at (x, y, z) projected into keyframe k of the launch (inv_pose: its inverse pose) and
// offered at its pixel.
template <bool kCandidatesOnly, bool kAdaptive = false>
LTR_DEV void exact_pair(float x, float y, float z, uint32_t i, uint32_t k, const double* __restrict__ inv_pose, const double* __restrict__ ext,
                        int ext_identity, int order, const ImgShape& g, const uint32_t* __restrict__ scan_rimg, float thres,
                        uint64_t* __restrict__ win, int shortcut, unsigned* n_atomics) {
    float lx, ly, lz;
    map_to_sensor(inv_pose, ext, ext_identity, order, x, y, z, &lx, &ly, &lz);
    const Sph s = cart2sph(lx, ly, lz);
    int r, c;
    pixel_index(s, g, &r, &c);
    offer<kCandidatesOnly, kAdaptive>(win, (size_t)k * g.rows * g.cols + (size_t)r * g.cols + c, s.r, i, scan_rimg, thres, shortcut, n_atomics);
}

// Kind A: pixel index known to be right, only the exact range is needed (double transform + sqrt): ~60 instructions.
template <bool kCandidatesOnly, bool kAdaptive = false>
LTR_DEV void exact_range_pair(const PtrView& map, uint64_t e, const double* __restrict__ poses, int kf0, const double* __restrict__ ext,
                              int ext_identity, int order, uint32_t npx, const uint32_t* __restrict__ scan_rimg, float thres,
                              uint64_t* __restrict__ win, int shortcut, unsigned* n_atomics) {
    const uint32_t i = (uint32_t)(e >> 32), pxl = ((uint32_t)e >> 14) & 0x3ffffu, k = (uint32_t)e & 0x3fffu;
    float lx, ly, lz;
    map_to_sensor(poses + (size_t)(kf0 + k) * 24, ext, ext_identity, order, map.x[i], map.y[i], map.z[i], &lx, &ly, &lz);
    const float r = __fsqrt_rn(fa(fa(fm(lx, lx), fm(ly, ly)), fm(lz, lz)));   // == cart2sph().r
    offer<kCandidatesOnly, kAdaptive>(win, (size_t)k * npx + pxl, r, i, scan_rimg, thres, shortcut, n_atomics);
}

// Kind B: nothing is known (pixel near a rounding boundary, degenerate geometry, keyframe without fast constants): the full reference
// arithmetic, as in map_project_kernel.
template <bool kCandidatesOnly, bool kAdaptive = false>
__device__ __noinline__ void exact_full_pair(const PtrView& map, uint64_t e, const double* __restrict__ poses, int kf0,
                                             const double* __restrict__ ext, int ext_identity, int order, const ImgShape& g,
                                             const uint32_t* __restrict__ scan_rimg, float thres, uint64_t* __restrict__ win, int shortcut,
                                             unsigned* n_atomics) {
    const uint32_t i = (uint32_t)(e >> 32), k = (uint32_t)e & 0x3fffu;
    exact_pair<kCandidatesOnly, kAdaptive>(map.x[i], map.y[i], map.z[i], i, k, poses + (size_t)(kf0 + k) * 24, ext, ext_identity, order, g, scan_rimg, thres,
                                win, shortcut, n_atomics);
}

}  // namespace ltr
#include "project_cull.cuh"
namespace ltr {

// the same pointer, opaque to the compiler: indexing it costs one IMAD.WIDE instead of re-deriving the 64-bit element offset per load
LTR_DEV const uint32_t* opaque_ptr(const uint32_t* p) { asm("mov.b64 %0, %0;" : "+l"(p)); return p; }

constexpr int kFastThreads = 256;
constexpr int kFastCtasPerSm = 3;   // 80 registers per thread: the per-keyframe and image constants stay in registers across the 4 points of a step
// The guard-padded variant (HD / revert / PD passes) fits 64 registers without spills and runs 4 CTAs per SM: the kernel waits on its
// (mostly L2) image gathers rather than on instruction issue, and the fourth CTA hides more of that latency (DESIGN.md 4.1)
constexpr int kFastCtasPerSmPad = 4;
constexpr int kFastPts = 4;      // map points per thread (registers); lane l of a warp holds points tile * 128 + 32 j + l
constexpr int kQueueCap = 160;   // per warp and kind: < 32 left over + 4 * 32 pushed per keyframe step
constexpr int kFastMaxBatch = 32;   // keyframes per launch: their constants travel as a kernel parameter (constant bank)

// Per-keyframe constants of one launch, passed BY VALUE: the kernel reads them from the constant bank with warp-uniform addresses, so
// they live in uniform registers / constant operands of the FFMAs instead of 16 vector registers and 4 shared-memory loads per step.
struct KfBatch { float kf[kFastMaxBatch][16]; };

// `test_img` (u32 per pixel, float bits):
//   kCandidatesOnly: the scan range image with "no return" pixels replaced by -inf when FastCfg::empty_scan_shortcut (built by
//       scan_test_image_kernel): a pair can only matter if  scan - range > thres  for SOME range within the margin.
//       kAdaptive (threshold t = fl(c s) per pixel, c in `thres`): the image holds v = fl_up(s - fl(c s)) >= s - t instead of s, and the
//       certainty threshold is 0.  A candidate has fl(s - rho) > t, hence s - rho > t (t is a float and rounding is monotone), hence
//       v - rho > 0: the test of the constant threshold with (v, 0) in place of (s, thres) keeps every candidate.  Rounding v up makes
//       the rounding bound delta of fl(s - t) zero, for every pixel: a pixel without a return (s = 10000, no shortcut) included.
//   otherwise: the running minimum `approx_min` itself.
// `approx_min` (u32 per pixel, float bits, initialised to +inf): running minimum of the APPROXIMATE ranges of the pairs that were queued
// for the pixel.  A pair whose approximate range exceeds it by more than twice the range margin is provably farther than an
// already-queued pair and cannot win the pixel, so it is dropped without exact arithmetic.
//
// Hot loop (profiles/sass_mix.py prints its SASS mix): the common "no effect" path is one straight line per point -- transform,
// azimuth, ranges, elevation, certainty, and (guard-padded variant) one IMAD + one unsigned min for the gather index: 64 instructions
// per point, 44 of them FP32 arithmetic -- and rare pairs reserve a queue slot with a shared-memory atomic (no ballots on the common
// path).  Measured on an H100, the kernel waits on its image gathers more than on instruction issue: cutting that line from 76 to 64
// instructions alone did not shorten it; the fourth CTA per SM that the 64 registers of the padded variant allow did (DESIGN.md 4.1).
// Deferred true-minimum mode (kDeferred; ND pass and visible-point extraction).  The pixel winner is the point of minimum EXACT
// range (lowest index on ties); an approximate range is within `band/2 = m_r_abs + m_r_rel r` of the exact one.  Instead of sending
// every running minimum through the exact arithmetic (on Morton-ordered surface patches that was 44 % of all pairs), the scan only
// maintains, per pixel, the pair of smallest APPROXIMATE range (`best`, 64-bit atomicMin of range bits | index) and appends to a
// small overflow list every pair that is within `band` of the best known at its time without becoming the best, as well as a
// displaced best that is within `band` of its successor.  `best` only decreases, so every point whose approximate range is within
// `band` of the FINAL best -- a superset of the points that can be the exact winner -- is either the final best or on the list.
// deferred_resolve_kernel then evaluates exactly the final best of every pixel and the list entries (a few per cent of a pixel
// count instead of tens of per cent of all pairs).  A full list sets `overflow_count` beyond the capacity; the host then repeats the
// call with the immediate mode.
// With `order`, the warps claim the tiles near to far from the keyframes of the launch, so that `best` holds near surfaces before
// the far tiles arrive: a pixel's running minimum drops fewer times, so fewer pairs issue the returning atomic.  The order cannot
// change a result: the argument above holds for any order in which the pairs arrive (DESIGN.md 4.1).
struct DeferredArgs {
    unsigned long long* best;      // [keyframes in launch][npx], initialised to ~0
    unsigned long long* list;      // overflow entries: q_pack(index, pixel, keyframe)
    unsigned int* count;           // entries appended by the current launch (may exceed capacity)
    unsigned int* overflow;        // set to 1 when that happened (sticky over the launches of a call)
    unsigned int capacity;
    const unsigned long long* order;   // tile claim order (low 32 bits: tile index), or nullptr: map order
};

// Ball subset of the map (ltr_remove_pass_ball, DESIGN.md 4.3): keyframe k of a launch sees only the map points with
// fl(fl(dx dx + dy dy) + dz dz) < r2, d = fl(p - c_k), c_k the f32 translation of its pose.  Per launch, ball_tile_list_kernel classifies
// every 128-point tile against every keyframe of the launch (`out`: no point of the tile is a member, `in`: every point is) and lists
// the tiles that are not `out` in all of them; map_project_fast_kernel<..., kBall> claims only the listed tiles.
struct BallArgs {
    const float4* centre;      // [keyframes in launch]: c_k (w unused); nullptr: no ball
    const uint32_t* out_mask;  // [tile]: bit k = no point of the tile is in ball k
    const uint32_t* in_mask;   // [tile]: bit k = every point of the tile is in ball k
    const uint32_t* list;      // tiles to project, in any order
    const unsigned int* count; // number of listed tiles (device-side, written by ball_tile_list_kernel)
    float r2;
};

// the exact membership test of the contract: FLANN's L2_Simple distance in f32 without contraction, strictly below r2 (NaN: not a member)
LTR_DEV bool ball_member(float x, float y, float z, float4 c, float r2) {
    const float dx = __fsub_rn(x, c.x), dy = __fsub_rn(y, c.y), dz = __fsub_rn(z, c.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)) < r2;
}

// One warp per tile, lane k against ball k of the launch (DESIGN.md 4.3 derives the slack).  With the tile sphere (c, rho) and
// D = |c - c_k| evaluated in double, every point p of the tile has D - rho <= |p - c_k| <= D + rho, and the f32 d2 of the contract is
// within 5u (u = 2^-24) relative of |p - c_k|^2 (no underflow matters once r2 >= 2^-100).  The double evaluation is within 1e-15 relative.
//   out: D - rho > 0 and (D - rho)^2 >= r2 (1 + 2^-20)  =>  d2 >= r2 (1 + 2^-20)(1 - 5u - 1e-15) > r2
//   in : (D + rho)^2 <= r2 (1 - 2^-20), every point of the tile finite  =>  d2 <= r2 (1 - 2^-20)(1 + 5u + 1e-15) < r2
// Outside r2 in [2^-100, FLT_MAX] nothing is classified, and every point takes the exact test.  Listed: every tile whose `out` mask is not
// all nb keyframes; the pairs of its `out` bits are counted as culled pairs (counters[3]), those of an unlisted tile too.
__global__ void __launch_bounds__(256) ball_tile_list_kernel(const float4* __restrict__ tiles, const uint8_t* __restrict__ tile_nonfinite,
                                                             long long ntiles, BallArgs ba, int nb, uint32_t* __restrict__ out_mask,
                                                             uint32_t* __restrict__ in_mask, uint32_t* __restrict__ list,
                                                             unsigned int* __restrict__ count, unsigned long long* __restrict__ counters) {
    const long long tile = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (tile >= ntiles) return;
    const unsigned lane = threadIdx.x & 31;
    bool out = false, in = false;
    const double r2 = (double)ba.r2;
    if ((int)lane < nb && r2 >= 0x1p-100 && r2 <= 3.4028234663852886e38) {
        const float4 t = tiles[tile], c = ba.centre[lane];
        const double dx = (double)t.x - (double)c.x, dy = (double)t.y - (double)c.y, dz = (double)t.z - (double)c.z;
        const double D = sqrt(dx * dx + dy * dy + dz * dz), rho = (double)t.w;
        const double lo = D - rho, hi = D + rho;
        out = lo > 0.0 && lo * lo >= r2 * (1.0 + 0x1p-20);   // NaN: false
        in = !tile_nonfinite[tile] && hi * hi <= r2 * (1.0 - 0x1p-20);
    }
    const unsigned om = __ballot_sync(0xffffffffu, out), im = __ballot_sync(0xffffffffu, in);
    if (lane == 0) {
        out_mask[tile] = om;
        in_mask[tile] = im;
        const unsigned all = nb >= 32 ? 0xffffffffu : (1u << nb) - 1u;
        if (om != all) list[atomicAdd(count, 1u)] = (uint32_t)tile;
        if (om && counters) atomicAdd(&counters[3], (unsigned long long)__popc(om) * (unsigned long long)kTilePts);
    }
}

// 1 per tile that holds a non-finite coordinate (such a point is never a ball member, and the tile sphere does not bound it); zeroed before
__global__ void __launch_bounds__(256) tile_nonfinite_kernel(PtrView map, uint8_t* __restrict__ tile_nonfinite) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= map.n) return;
    if (!(isfinite(map.x[i]) && isfinite(map.y[i]) && isfinite(map.z[i]))) tile_nonfinite[i / kTilePts] = 1;
}

template <bool kCandidatesOnly, bool kElDirect, bool kDeferred = false, bool kPad = false, bool kAdaptive = false, bool kBall = false>
__global__ void __launch_bounds__(kFastThreads, kPad ? kFastCtasPerSmPad : kFastCtasPerSm) map_project_fast_kernel(PtrView map, const __grid_constant__ KfBatch kb, const double* __restrict__ poses,
                                                                        int kf0, int nb, const double* __restrict__ ext, int ext_identity, int order,
                                                                        ImgShape g, const __grid_constant__ FastCfg fc, const uint32_t* __restrict__ scan_rimg,
                                                                        const uint32_t* __restrict__ test_img, float thres,
                                                                        uint64_t* __restrict__ win, uint32_t* __restrict__ approx_min,
                                                                        CullArgs ca, unsigned long long* __restrict__ counters,
                                                                        unsigned int* __restrict__ work_counter, DeferredArgs da, BallArgs ba) {
    // kPad (scan-minus-map, short elevation path, 360 degree field of view): the test image is guard-padded (FastCfg::pad_*), so the
    // gather needs no index clamp
    static_assert(!kPad || (kCandidatesOnly && kElDirect && !kDeferred), "the padded test image exists for the scan-minus-map short path only");
    static_assert(!kAdaptive || (kCandidatesOnly && !kDeferred), "the true minimum does not depend on the threshold");
    // kBall: the warps claim the tiles of ba.list (ball_tile_list_kernel); a point outside ball k is absent from keyframe k -- no
    // certainty decision, queue entry, atomic or deferred-list entry.  The claim order cannot change a result (DESIGN.md 4.3).
    extern __shared__ uint64_t s_queues[];
    const int warp = threadIdx.x >> 5;
    uint64_t* s_qa = s_queues + warp * (2 * kQueueCap);
    uint64_t* s_qb = s_qa + kQueueCap;
    __shared__ int s_cnt[kFastThreads / 32][2];
    __shared__ unsigned s_stat[kFastThreads / 32][3];   // per warp: pairs through the exact-range / full exact path, culled (tile, keyframe) tests
    if ((threadIdx.x & 31) < 2) s_cnt[warp][threadIdx.x & 31] = 0;
    if ((threadIdx.x & 31) < 3) s_stat[warp][threadIdx.x & 31] = 0;
    __syncthreads();
    const unsigned lane = threadIdx.x & 31;
    const uint32_t npx = (uint32_t)(g.rows * g.cols);
    const int hi_c = g.cols - 1, hi_r = g.rows - 1;
    const float kMagic = 12582912.0f;            // 1.5 * 2^23: v + kMagic has the nearest integer in its low mantissa bits
    // kAdaptive: `thres` is the coefficient c, and the test image holds an upper bound of s - fl(c s), so that the certainty threshold is 0
    const float thr_lo = (kAdaptive ? 0.0f : thres) - fc.m_r_abs;
    unsigned n_atomics = 0;
#ifdef LTR_PROBE_NOMAYBE
    unsigned n_nomaybe = 0;
#endif
    // Persistent warps: each warp claims 128-point tiles from a global counter until the map is exhausted, so warps whose
    // tiles are culled in many keyframes do not leave issue slots idle while their CTA-mates finish.
    const long long total_tiles = (map.n + (32 * kFastPts) - 1) / (32 * kFastPts);
    for (;;) {
    unsigned tile_u = 0;
    if (lane == 0) tile_u = atomicAdd(work_counter, 1u);
    tile_u = __shfl_sync(0xffffffffu, tile_u, 0);
    if (kBall ? tile_u >= *ba.count : (long long)tile_u >= total_tiles) break;
    const long long tile = kBall ? (long long)ba.list[tile_u] : (kDeferred && da.order) ? (long long)(uint32_t)da.order[tile_u] : (long long)tile_u;
    const int64_t base = (int64_t)tile * (32 * kFastPts) + lane;
    // map index of the lane's point j, and the push of its pair with keyframe k onto the full exact queue.  Recomputed at each use: caching
    // the indices across the keyframe loop would cost the padded variant its 64-register bound.
    const auto point_index = [&](int j) { return (uint32_t)(base + j * 32 < map.n ? base + j * 32 : map.n - 1); };
    const auto push_full = [&](int j, int k) { s_qb[atomicAdd(&s_cnt[warp][1], 1)] = q_pack(point_index(j), 0u, (uint32_t)k); };
    float px_[kFastPts], py_[kFastPts], pz_[kFastPts];
#pragma unroll
    for (int j = 0; j < kFastPts; ++j) {
        // the last tile re-processes point n-1 in its padding lanes: harmless (atomicMin of an identical key)
        const int64_t i = min(base + (int64_t)j * 32, map.n - 1);
        px_[j] = map.x[i]; py_[j] = map.y[i]; pz_[j] = map.z[i];
    }
    // Tile culling (project_cull.cuh): lane l tests this 128-point tile against keyframe l of the launch; the ballot is the
    // set of keyframes in which no point of the tile can be a candidate -- those iterations of the k loop are skipped.
    // kBall: the keyframes whose ball holds no point of the tile are skipped like culled ones (their pairs were counted by the list kernel)
    unsigned cull_mask = kBall ? ba.out_mask[tile] : 0u;
    const unsigned ball_in = kBall ? ba.in_mask[tile] : 0u;
    if (kCandidatesOnly && ca.enabled) {
        const float4 t = ca.tiles[tile];
        const bool c = ((int)lane < nb) && (!kBall || !((cull_mask >> lane) & 1u)) && tile_culled<kAdaptive>(kb.kf[lane], t, fc, g, ca, (int)lane, thres);
        const unsigned m = __ballot_sync(0xffffffffu, c);
        cull_mask |= m;
        if (lane == 0) s_stat[warp][2] += __popc(m);
    }
    for (int k = 0; k < nb; ++k) {                    // a plain counted loop: k stays provably warp-uniform, so kb.kf[k] is read with LDCU
        if ((cull_mask >> k) & 1u) continue;         // warp-uniform (ballot)
        const float* __restrict__ kf = kb.kf[k];
        // kBall: the membership of the thread's points in ball k (all members when the tile's `in` bit is set; warp-uniform branch)
        bool in_[kFastPts];
#pragma unroll
        for (int j = 0; j < kFastPts; ++j) in_[j] = true;
        if (kBall && !((ball_in >> k) & 1u)) {
            const float4 bc = ba.centre[k];
#pragma unroll
            for (int j = 0; j < kFastPts; ++j) in_[j] = ball_member(px_[j], py_[j], pz_[j], bc, ba.r2);
        }
        if (kf[15] == 0.0f) {                         // warp-uniform: no fast constants (non-rigid pose or extrinsic) -> all pairs exact
#pragma unroll
            for (int j = 0; j < kFastPts; ++j) if (in_[j]) push_full(j, k);
        } else {
        // this keyframe's images (kPad: the padded test image)
        const uint32_t* __restrict__ test_k = kDeferred ? nullptr : kPad ? opaque_ptr(test_img + (uint32_t)(k * fc.pad_npx)) : test_img + (size_t)k * npx;
        uint32_t* __restrict__ amin_k = kDeferred ? nullptr : approx_min + (size_t)k * npx;
        unsigned long long* __restrict__ best_k = kDeferred ? da.best + (size_t)k * npx : nullptr;
        // Phase 1, branch-free: project the thread's points and ISSUE all their image gathers, so that the (mostly L2) latencies of
        // the four loads overlap instead of being paid one after the other behind a branch each.
        float fr_[kFastPts], tv_[kFastPts];
        uint32_t pxl_[kFastPts];   // kPad: bits of the float index, else the pixel
        bool certain_[kFastPts];
#pragma unroll
        for (int j = 0; j < kFastPts; ++j) {
            const FastProj f = fast_project<kElDirect>(kf, px_[j], py_[j], pz_[j]);
            const float vcol = __fmaf_rn(f.az, fc.col_scale, fc.col_off);
            const float vrow = __fmaf_rn(f.el, fc.neg_row_scale, fc.row_off);
            const float yc = __fadd_rn(vcol, kMagic), yr = __fadd_rn(vrow, kMagic);
            const float dc = fabsf(__fsub_rn(vcol, __fsub_rn(yc, kMagic)));   // distance to the nearest integer (NaN stays NaN)
            const float dr = fabsf(__fsub_rn(vrow, __fsub_rn(yr, kMagic)));
            // certain <=> both coordinates are farther than their margin from a rounding boundary (false for NaN), and the azimuth is not
            // within half a pixel of +-pi.  The seam rule: a sensor-frame y that is zero or within the transform error of zero may have the
            // other sign in the reference, which then puts the pair on the other side of the seam (column 0 <-> C - 1 at 360 degrees, the
            // opposite clamped edge otherwise) although the fast column looks certain.  The column margin bounds the azimuth error modulo
            // 2 pi, so such a pair's fast azimuth is within its margin of +-pi, and a certain pair's margin is below half a pixel: the band
            // holds every such pair, which then takes the full exact path.  NaN compares false.  kPad keeps its sentinel columns instead.
            certain_[j] = (__fmaf_rn(fc.m_col_b, f.rho_inv_r, dc) < fc.lim_c) & (dr < fc.lim_r) & (kPad || fabsf(f.az) < fc.az_seam_lim);
            fr_[j] = f.r;
            if (kPad) {
                // guard-padded test image (scan_test_image_kernel): the rounded row n_r = yr - kMagic lies in [-g, R - 1 + g] and the rounded
                // column in [0, C] (FastCfg::pad_*); the guard rows replicate the first / last row, which pixel_index clamps to.  Columns 0 and C
                // hold +inf: there the azimuth is within half a pixel of +-pi, and a sensor-frame y that is zero or within the transform error
                // of it may have the other sign in the reference, which puts the pair on the other side of the seam (column 0 <-> C - 1) even
                // though the column looks certain.  +inf makes every such pair `maybe`, and the maybe branch sends it to the full exact path.
                // The bits of yr and yc are 0x4B400000 + n_r and 0x4B400000 + n_c, so bits(yr) (C + 1) + bits(yc) - pad_bias is, modulo 2^32,
                // the padded index (n_r + g)(C + 1) + n_c: one IMAD.  One unsigned min keeps every other value inside the image: a NaN, or an
                // azimuth that left [-pi, pi] (denormal sensor-frame coordinates, rcp -> inf); neither pair is certain.
                const uint32_t pp = min(__float_as_uint(yr) * fc.pad_w + __float_as_uint(yc) - fc.pad_bias, fc.pad_last);
                pxl_[j] = pp;
                tv_[j] = __uint_as_float(__ldg(test_k + pp));   // one IMAD.WIDE.U32 from the keyframe's base
            } else {
                const int c = min(max(__float_as_int(yc) - 0x4B400000, 0), hi_c);   // NaN -> some in-range pixel; such a pair is never "certain"
                const int r = min(max(__float_as_int(yr) - 0x4B400000, 0), hi_r);
                pxl_[j] = (uint32_t)(r * g.cols + c);
                // unconditional: the index is always inside the image (deferred mode: the range word of the pixel's best pair)
                tv_[j] = kDeferred ? __uint_as_float(reinterpret_cast<const uint32_t*>(best_k)[2 * pxl_[j] + 1]) : __uint_as_float(test_k[pxl_[j]]);
            }
        }
        // Phase 2: decide.  Almost every pair ends at the first comparison.
        if (kDeferred) {
            // 2a: issue the atomics of all four points back to back (their round trips overlap), 2b: use what they returned.
            // (Reducing the running minima of a pixel inside the warp first -- match.any on the pixel, redux.min -- was measured slower:
            // the match costs more than the atomics it saves.)
            unsigned long long old_[kFastPts];
            float rwin_[kFastPts];
            bool enter_[kFastPts], lead_[kFastPts];
#pragma unroll
            for (int j = 0; j < kFastPts; ++j) {
                const float fr = fr_[j], tv = tv_[j];
                // tv = approximate range of the pixel's best pair as read in phase 1 (all-ones bits = NaN while the pixel is empty;
                // every comparison is written so that NaN means "consider the pair")
                enter_[j] = in_[j] && certain_[j] && !(fr > __fadd_rn(tv, __fmaf_rn(fc.mr2_rel, fr, fc.mr2_abs)));
                lead_[j] = enter_[j] && !(fr >= tv);             // looks like a new best
                old_[j] = 0ull; rwin_[j] = tv;
                if (lead_[j]) {
                    old_[j] = atomicMin(&best_k[pxl_[j]], ((unsigned long long)__float_as_uint(fr) << 32) | point_index(j));
                    ++n_atomics;
                }
            }
#pragma unroll
            for (int j = 0; j < kFastPts; ++j) {
                if (enter_[j]) {
                    const float fr = fr_[j];
                    const unsigned long long v = ((unsigned long long)__float_as_uint(fr) << 32) | point_index(j);
                    // not the group's representative (or not better than what was read): v is a candidate that loses to a pair of range rwin_
                    unsigned long long loser = v;
                    float r_win = rwin_[j];
                    if (lead_[j]) {
                        if (v < old_[j]) { loser = old_[j]; r_win = fr; }                        // v is the best now; the displaced pair may still matter
                        else r_win = __uint_as_float((uint32_t)(old_[j] >> 32));                 // somebody nearer got there first
                    }
                    const float r_los = __uint_as_float((uint32_t)(loser >> 32));
                    if (loser != ~0ull && !(r_los > __fadd_rn(r_win, __fmaf_rn(fc.mr2_rel, r_los, fc.mr2_abs)))) {
                        const unsigned slot = atomicAdd(da.count, 1u);
                        if (slot < da.capacity) da.list[slot] = q_pack((uint32_t)loser, pxl_[j], (uint32_t)k);
                    }
                } else if (in_[j] && !certain_[j]) {
                    push_full(j, k);
                }
            }
        } else {
#ifdef LTR_PROBE_NOMAYBE
        bool any_maybe = false;
#endif
#pragma unroll
        for (int j = 0; j < kFastPts; ++j) {
            const float fr = fr_[j], tv = tv_[j];
            if (!in_[j]) continue;                   // kBall: not in this keyframe's ball
            if (certain_[j]) {
                bool maybe;
                if (kCandidatesOnly) maybe = !(__fmaf_rn(fr, fc.rel_m1, tv) < thr_lo);   // scan - r + m_rel r >= thres - m_abs for some range within the margin
                else maybe = !(fr > __fadd_rn(tv, __fmaf_rn(fc.mr2_rel, fr, fc.mr2_abs)));   // not provably farther than an already-queued pair
#ifdef LTR_PROBE_NOMAYBE
                any_maybe |= maybe;
#endif
                if (maybe) {
                    uint32_t pxl = pxl_[j];
                    bool seam = false;
                    if (kPad) {   // padded index -> pixel of the unpadded images (approx_min, queue entries, exact path)
                        const uint32_t rp = pxl / (uint32_t)(g.cols + 1);
                        const int col = (int)(pxl - rp * (uint32_t)(g.cols + 1));
                        seam = (col == 0) | (col == g.cols);   // +inf in the test image: the reference may put the pair across the seam
                        pxl = (uint32_t)(min(max((int)rp - fc.pad_g, 0), hi_r) * g.cols + min(col, hi_c));
                    }
                    if (kPad && seam) {
                        push_full(j, k);
                        continue;
                    }
                    bool push = true;
                    if (kCandidatesOnly) {
                        const float cur = __uint_as_float(amin_k[pxl]);
                        push = !(fr > __fadd_rn(cur, __fmaf_rn(fc.mr2_rel, fr, fc.mr2_abs)));
                        if (push && fr < cur) atomicMin(&amin_k[pxl], __float_as_uint(fr));
                    } else if (fr < tv) atomicMin(&amin_k[pxl], __float_as_uint(fr));
                    if (push) s_qa[atomicAdd(&s_cnt[warp][0], 1)] = q_pack(point_index(j), pxl, (uint32_t)k);
                }
            } else {
                push_full(j, k);
            }
        }
#ifdef LTR_PROBE_NOMAYBE
        // diagnostic build of profiles/hd_pass_probe.py only: counts the non-culled (tile, keyframe) iterations in which no lane took the
        // `maybe` branch -- what any tile-level cull could still remove -- and reports them in place of the atomics count
        if (!__any_sync(0xffffffffu, any_maybe) && lane == 0) ++n_nomaybe;
#endif
        }
        }  // keyframe with fast constants
        __syncwarp();
        int qa = *(volatile int*)&s_cnt[warp][0];
        int qb = *(volatile int*)&s_cnt[warp][1];
        if ((qa | qb) >= 32) {   // warp-uniform
            while (qa >= 32) {
                qa -= 32;
                const uint64_t e = s_qa[qa + lane];
                exact_range_pair<kCandidatesOnly, kAdaptive>(map, e, poses, kf0, ext, ext_identity, order, npx, scan_rimg, thres, win, fc.empty_scan_shortcut, &n_atomics);
                if (lane == 0) s_stat[warp][0] += 32;
            }
            while (qb >= 32) {
                qb -= 32;
                const uint64_t e = s_qb[qb + lane];
                exact_full_pair<kCandidatesOnly, kAdaptive>(map, e, poses, kf0, ext, ext_identity, order, g, scan_rimg, thres, win, fc.empty_scan_shortcut, &n_atomics);
                if (lane == 0) s_stat[warp][1] += 32;
            }
            __syncwarp();
            if (lane == 0) { s_cnt[warp][0] = qa; s_cnt[warp][1] = qb; }
            __syncwarp();
        }
    }
    }  // persistent tile loop
    const int qa = *(volatile int*)&s_cnt[warp][0], qb = *(volatile int*)&s_cnt[warp][1];
    if ((int)lane < qa) {
        exact_range_pair<kCandidatesOnly, kAdaptive>(map, s_qa[lane], poses, kf0, ext, ext_identity, order, npx, scan_rimg, thres, win, fc.empty_scan_shortcut, &n_atomics);
    }
    if ((int)lane < qb) {
        exact_full_pair<kCandidatesOnly, kAdaptive>(map, s_qb[lane], poses, kf0, ext, ext_identity, order, g, scan_rimg, thres, win, fc.empty_scan_shortcut, &n_atomics);
    }
    // statistics: [0] pairs through the exact-range path (deferred mode: deferred_resolve_kernel adds the list entries), [1] atomics on
    // the winner image (deferred mode: plus those on `best`), [2] pairs through the full exact path, [3] culled pairs
#ifdef LTR_PROBE_NOMAYBE
    n_atomics = n_nomaybe;
#endif
    for (int o = 16; o > 0; o >>= 1) {
        n_atomics += __shfl_down_sync(0xffffffffu, n_atomics, o);
    }
    if (lane == 0 && counters) {
        const unsigned n_a = s_stat[warp][0] + (unsigned)qa, n_b = s_stat[warp][1] + (unsigned)qb, n_culled = s_stat[warp][2];
        atomicAdd(&counters[0], (unsigned long long)n_a); atomicAdd(&counters[1], (unsigned long long)n_atomics); atomicAdd(&counters[2], (unsigned long long)n_b);
        if (n_culled) atomicAdd(&counters[3], (unsigned long long)n_culled * (32ull * kFastPts));   // pairs skipped by tile culling
    }
}

// Deferred true-minimum mode, second half: the exact (range, index) key of the final best pair of every pixel and of every list entry
// goes into the winner image with the same 64-bit atomicMin as everywhere else.
__global__ void __launch_bounds__(256) deferred_resolve_kernel(PtrView map, const double* __restrict__ poses, int kf0, int nb, const double* __restrict__ ext,
                                                               int ext_identity, int order, uint32_t npx, DeferredArgs da, uint64_t* __restrict__ win,
                                                               unsigned long long* __restrict__ counters) {
    const int64_t total = (int64_t)nb * npx;
    const unsigned n_list = min(*da.count, da.capacity);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        if (*da.count > da.capacity) *da.overflow = 1u;
        if (counters) atomicAdd(&counters[0], (unsigned long long)*da.count);   // list appends: pairs through the exact-range path
    }
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total + n_list; t += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long e;
        if (t < total) {
            const unsigned long long b = da.best[t];
            if (b == ~0ull) continue;
            e = q_pack((uint32_t)b, (uint32_t)(t % npx), (uint32_t)(t / npx));
        } else e = da.list[t - total];
        unsigned n_atomics = 0;
        exact_range_pair<false>(map, e, poses, kf0, ext, ext_identity, order, npx, nullptr, 0.0f, win, 0, &n_atomics);
    }
}

}  // namespace ltr
