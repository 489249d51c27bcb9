// libltr_b200.so -- per-keyframe kNN set difference, the primitive of LT-map change composition and map rollback (DESIGN.md §5.3).
//
// ltr_knn_split_per_keyframe: every point of keyframe k of `query` is tested against the points of keyframe k of `target` only, with
// the rule of every kNN decision (ref_math.cuh, TopK): near iff |(float)(sum_double of its k smallest L2_Simple squared distances) /
// float(k)| < thr; a target keyframe of 0 < n < k points contributes all n and the sum is still divided by k (knn_label_all).  Unlike
// the other kNN entry points an empty target keyframe is not an error: its query points are all "far" (an empty per-keyframe delta is the
// common case of composition).
//
// Search.  One sparse grid level (sparse_grid.cuh, built by scanside.cu's build_level) keyed by (keyframe of the launch, cell) holds the
// targets of the launch's keyframes.  One thread per query point walks the 27 cells around its own cell in its own keyframe with the
// dense grid's walk (ref_math.cuh, knn_label_27: k smallest distances in registers, early exit on "near"), one sparse row lookup
// (sparse_grid.cuh, row_points) per row of three cells.
// Why 27 cells are exact.  Let c = 1 / inv_cell be the cell side the indices are computed with and B(1) = ((1 - 2^-6) c)^2 (1 - 2^-20)
// (shell_bound).  sparse_grid.cuh's header proves that every target point outside the 27-cell block has a computed distance STRICTLY
// greater than B(1).  The host picks c so that B(1) >= k thr (1 + 2^-21), evaluated in double (relative error < 2^-50, far inside the
// margin).  Let D_1 <= ... <= D_k be the true k smallest computed distances over the whole target keyframe (it has >= k points here).
//  * D_k <= B(1): every point at distance <= D_k lies in the block, so the block's k smallest are the true ones as a multiset, and so
//    are the sum and the mean.
//  * D_k > B(1): the true double sum S of non-negative terms in ascending order is >= D_k > k thr (1 + 2^-21); its f32 rounding is
//    >= S (1 - 2^-24) > k thr, so the f32 quotient by the exact float(k) is >= thr (division by an exact k and rounding are monotone and
//    thr is a float): the truth is "far".  The block agrees: with fewer than k block points it says "far"; otherwise its k smallest are
//    element-wise >= D_1..D_k (a subset), so its mean is >= the true mean >= thr.  An overflowed +inf term gives +inf, "far", on both sides.
// Keyframes with 0 < n < k target points skip the grid and sum all n distances by brute force; empty target keyframes write "far".
// Launches: keyframes go through in launches of at most 8192 keyframes (the level's segment bits) and at most LTR_DELTA_CHUNK_POINTS query +
// target points (environment; default 2^24, one keyframe at least).  Cells grow by 1.25x from the reach above until the launch's target
// extent fits in 2^17 - 1 cells per axis (as build_grid grows its dense grid).
// Memory: one flag byte per query point for the call; per launch the level (28 B per target point, plus 32 B per target point of sort
// scratch while it is built) and two offset arrays; the outputs (16 B per query point together) come from split_scanset_by_flag.  All
// scratch is returned before the call ends.
#include "ltr_internal.cuh"
#include "ref_math.cuh"
#include "device_util.cuh"
#include "sparse_grid.cuh"
#include <algorithm>
#include <cmath>

namespace ltr {

namespace {

constexpr int64_t kChunkPoints = (int64_t)1 << 24;

// 1 = far, 0 = near for the query (qx, qy, qz) against segment seg of the level (a target keyframe of >= k points)
template <int KT>
__device__ __forceinline__ uint8_t grid_label(const Level& L, int seg, float qx, float qy, float qz, int k, float thr) {
    int c[3];
    const float q[3] = {qx, qy, qz};
    // clamped to [-2, dim + 1]: a query's cell farther outside the box has no cell of the block either way
#pragma unroll
    for (int d = 0; d < 3; ++d) c[d] = (int)min(max(cell_index((double)q[d], L.origin[d], L.inv_cell), -2ll), (long long)L.dim[d] + 1);
    const uint32_t c0 = L.seg_first[seg], c1 = L.seg_first[seg + 1];
    auto rows = [&](int y, int z, int xa, int xb, uint32_t* s, uint32_t* e) { row_points(L, c0, c1, seg, xa, xb, y, z, s, e); };
    return knn_label_27<KT>(rows, L.pts, c[0], c[1], c[2], L.dim, qx, qy, qz, k, thr);
}

// The queries [qbase, qbase + m) of keyframes [kf0, kf0 + nkf): flag[i] = 1 (far) or 0 (near) against keyframe kf of the target.
// Segment j of L is keyframe kf0 + j.  sm_90a: 34-37 registers for k <= 4, 48 for k > 4, no spill; the minimum of 8 CTAs per SM does not
// bind at 48 registers, but with the bare bound ptxas gives k > 4 40 registers and a 12 B spill.
template <int KT>
__global__ void __launch_bounds__(128, 8) knn_split_kf_kernel(Level L, PtrView q, const int64_t* __restrict__ q_off, PtrView t,
                                                           const int64_t* __restrict__ t_off, int kf0, int nkf, int64_t qbase, int64_t m,
                                                           int k, float thr, uint8_t* __restrict__ flag) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const int64_t i = qbase + j;
    const int seg = find_kf(q_off + kf0, nkf, i);
    const int kf = kf0 + seg;
    const int64_t t0 = t_off[kf], nt = t_off[kf + 1] - t0;
    const float x = q.x[i], y = q.y[i], z = q.z[i];
    uint8_t f;
    if (nt == 0) f = 1;
    else if (nt < k) f = knn_label_all<KT>((int)nt, [&](int p) { return make_float4(t.x[t0 + p], t.y[t0 + p], t.z[t0 + p], 0.0f); }, x, y, z, k, thr);
    else f = grid_label<KT>(L, seg, x, y, z, k, thr);
    flag[i] = f;
}

int launch_split(ltr_ctx* ctx, int k, const Level& L, PtrView q, const int64_t* q_off, PtrView t, const int64_t* t_off, int kf0, int nkf,
                 int64_t qbase, int64_t m, float thr, uint8_t* flag) {
    if (m == 0) return LTR_OK;
    const unsigned nb = (unsigned)((m + 127) / 128);
    switch (k) {
#define LTR_DELTA_CASE(KK, KT) \
        case KK: knn_split_kf_kernel<KT><<<nb, 128, 0, ctx->stream>>>(L, q, q_off, t, t_off, kf0, nkf, qbase, m, k, thr, flag); break;
        LTR_DELTA_CASE(1, 1) LTR_DELTA_CASE(2, 2) LTR_DELTA_CASE(3, 3) LTR_DELTA_CASE(4, 4)
        default: knn_split_kf_kernel<kKnnMaxK><<<nb, 128, 0, ctx->stream>>>(L, q, q_off, t, t_off, kf0, nkf, qbase, m, k, thr, flag); break;
#undef LTR_DELTA_CASE
    }
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

// cell side for one launch: B(1) >= k thr (1 + 2^-21) (file header), grown until the target extent fits the level's index bits
double launch_cell(int k, float thr, const float mn[3], const float mx[3]) {
    const double need = (double)k * (double)thr * (1.0 + 0x1p-21);
    double cell = std::sqrt((double)k * (double)thr) * 1.02 + 1e-9;
    auto b1 = [](double c) { const double cc = 1.0 / (1.0 / c); const double r = (1.0 - 0x1p-6) * cc; return r * r * (1.0 - 0x1p-20); };
    while (b1(cell) < need) cell *= 1.01;
    for (;;) {
        int dmax = 0;
        for (int d = 0; d < 3; ++d) dmax = std::max(dmax, (int)std::min(std::floor(((double)mx[d] - (double)mn[d]) / cell) + 3.0, 2e9));
        if (dmax < kGridMaxDim) break;   // build_level's dim can exceed floor(ext / cell) + 3 by one rounding step
        cell *= 1.25;
    }
    return cell;
}

}  // namespace
}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_knn_split_per_keyframe(ltr_ctx* ctx, ltr_scanset query_h, ltr_scanset target_h, int32_t k, float thr, ltr_scanset* out_near,
                               ltr_scanset* out_far) {
    ApiTrace tr__(ctx, "ltr_knn_split_per_keyframe");
    if (!ctx) return LTR_ERR_INVALID;
    DevScanSet *qp, *tp;
    LTR_TRY(scanset_get(ctx, query_h, &qp));
    LTR_TRY(scanset_get(ctx, target_h, &tp));
    if (qp->K != tp->K) return fail(ctx, LTR_ERR_INVALID, "query has %d keyframes, target %d", qp->K, tp->K);
    if (k < 1 || k > kKnnMaxK) return fail(ctx, LTR_ERR_UNSUPPORTED, "k = %d outside [1, %d]", k, kKnnMaxK);
    if (!(thr > 0.0f) || !std::isfinite(thr)) return fail(ctx, LTR_ERR_INVALID, "threshold must be positive and finite");
    const DevScanSet Q = *qp, T = *tp;
    const int K = Q.K;
    float mn[3], mx[3];
    if (Q.pts.n > 0) LTR_TRY(finite_extent(ctx, Q.pts, "query", mn, mx));
    if (T.pts.n > 0) LTR_TRY(finite_extent(ctx, T.pts, "target", mn, mx));
    if (Q.pts.n == 0) {
        const std::vector<int64_t> off((size_t)K + 1, 0);
        ScanSetOwner o_near, o_far;
        if (out_near) LTR_TRY(scanset_new(ctx, off, &o_near));
        if (out_far) LTR_TRY(scanset_new(ctx, off, &o_far));
        if (out_near) *out_near = o_near.release();
        if (out_far) *out_far = o_far.release();
        return LTR_OK;
    }
    void* flags = nullptr;
    ScratchGuard g_flags(ctx, &flags);
    LTR_TRY(dev_alloc(ctx, &flags, (size_t)Q.pts.n));
    {
        // launches are planned on the query + target points of each keyframe
        std::vector<int64_t> both((size_t)K + 1);
        for (int j = 0; j <= K; ++j) both[(size_t)j] = Q.h_off[(size_t)j] + T.h_off[(size_t)j];
        int64_t max_chunk = 0;
        const std::vector<int> kf_cut = plan_keyframe_chunks(both, env_points("LTR_DELTA_CHUNK_POINTS", kChunkPoints, (int64_t)1 << 30),
                                                             kGridMaxSegments, &max_chunk);
        if (max_chunk >= ((int64_t)1 << 32)) return fail(ctx, LTR_ERR_UNSUPPORTED, "a keyframe of %lld points", (long long)max_chunk);
        void* offs = nullptr;
        ScratchGuard g_offs(ctx, &offs);
        LTR_TRY(dev_alloc(ctx, &offs, ((size_t)kGridMaxSegments + 1) * 8));
        int64_t* t_rel = (int64_t*)offs;
        for (size_t c = 0; c + 1 < kf_cut.size(); ++c) {
            const int kf0 = kf_cut[c], kf1 = kf_cut[c + 1], nkf = kf1 - kf0;
            const int64_t qbase = Q.h_off[(size_t)kf0], m = Q.h_off[(size_t)kf1] - qbase;
            if (m == 0) continue;
            const int64_t tbase = T.h_off[(size_t)kf0], nt = T.h_off[(size_t)kf1] - tbase;
            bool grid = false;
            for (int kf = kf0; kf < kf1; ++kf) grid |= T.h_off[(size_t)kf + 1] - T.h_off[(size_t)kf] >= k;
            LevelBuf lb;
            ScratchGuard g_level(ctx, &lb.block);
            if (grid) {
                DevCloud tc = T.pts;   // the launch's targets: a view with the set's component stride
                tc.base = T.pts.base + tbase;
                tc.n = nt;
                float tmn[3], tmx[3];
                LTR_TRY(minmax_xyz(ctx, tc, tmn, tmx));
                LTR_TRY(relative_offsets(ctx, T.d_off, kf0, nkf, t_rel));
                LTR_TRY(build_level(ctx, view(tc), t_rel, nkf, tmn, tmx, launch_cell(k, thr, tmn, tmx), true, &lb));
            }
            LTR_TRY(launch_split(ctx, k, lb.L, view(Q.pts), Q.d_off, view(T.pts), T.d_off, kf0, nkf, qbase, m, thr, (uint8_t*)flags));
        }
    }
    return split_scanset_by_flag(ctx, Q, (const uint8_t*)flags, out_near, out_far);
}

}  // extern "C"
