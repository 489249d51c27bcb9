// libltr_b200.so -- exact k-nearest-neighbour labelling on a dense uniform grid.
//
// Reference functions replaced:
//   Session::extractLowDynPointsViaKnnDiff / extractHighDynPointsViaKnnDiff   ltremovert/src/Session.cpp:393-427, 487-504
//   Session::partition{Low,High}DynamicPointsOfScanByKnn                      ltremovert/src/Session.cpp:537-607, 610-642
//   Session::removeWeakNDMapPointsHavingStrongNDInNear                        ltremovert/src/Session.cpp:452-484
// The reference queries pcl::KdTreeFLANN (FLANN KDTreeSingleIndex, L2_Simple<float>, exact) and tests
//   |(float)(sum_double of the k smallest SQUARED distances) / float(k)| < thr.
// Exactness of the grid search: every squared distance is >= 0, so a point can only be labelled "near" if all of its
// k nearest squared distances are < k*thr.  With cells of side >= sqrt(k*thr)*(1+slack) every such neighbour lies in the
// 27 cells around the query's cell; if one of the true k nearest lies outside them, its squared distance alone already
// exceeds k*thr and both searches label the point "far".  Squared distances are evaluated exactly as FLANN's L2_Simple:
// ((dx*dx) + dy*dy) + dz*dz in f32, dx = query - point, no FMA.
#include "ltr_internal.cuh"
#include "ref_math.cuh"
#include "device_util.cuh"
#include <algorithm>
#include <cmath>

namespace ltr {

__device__ __forceinline__ void cell_of(const KnnTarget& g, float x, float y, float z, int* cx, int* cy, int* cz) {
    *cx = (int)floor(((double)x - g.origin[0]) * g.inv_cell);
    *cy = (int)floor(((double)y - g.origin[1]) * g.inv_cell);
    *cz = (int)floor(((double)z - g.origin[2]) * g.inv_cell);
}

__global__ void __launch_bounds__(256) grid_count_kernel(PtrView t, KnnTarget g, uint32_t* __restrict__ cell_cnt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.n) return;
    int cx, cy, cz;
    cell_of(g, t.x[i], t.y[i], t.z[i], &cx, &cy, &cz);
    cx = min(max(cx, 0), g.dim[0] - 1); cy = min(max(cy, 0), g.dim[1] - 1); cz = min(max(cz, 0), g.dim[2] - 1);
    atomicAdd(&cell_cnt[((size_t)cz * g.dim[1] + cy) * g.dim[0] + cx], 1u);
}

__global__ void __launch_bounds__(256) grid_fill_kernel(PtrView t, KnnTarget g, uint32_t* __restrict__ cursor, float4* __restrict__ sorted) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.n) return;
    const float x = t.x[i], y = t.y[i], z = t.z[i];
    int cx, cy, cz;
    cell_of(g, x, y, z, &cx, &cy, &cz);
    cx = min(max(cx, 0), g.dim[0] - 1); cy = min(max(cy, 0), g.dim[1] - 1); cz = min(max(cz, 0), g.dim[2] - 1);
    const size_t c = ((size_t)cz * g.dim[1] + cy) * g.dim[0] + cx;
    const uint32_t slot = g.cell_start[c] + atomicAdd(&cursor[c], 1u);
    sorted[slot] = make_float4(x, y, z, 0.0f);
}

// decision "far" (1) or "near" (0) of (qx,qy,qz) from the 27 cells around its cell of the dense grid
template <int KT>
__device__ __forceinline__ uint8_t knn_label(const KnnTarget& t, float qx, float qy, float qz, int k, float thr) {
    int cx, cy, cz;
    cell_of(t, qx, qy, qz, &cx, &cy, &cz);
    auto rows = [&](int y, int z, int x0, int x1, uint32_t* s, uint32_t* e) {
        const size_t row = ((size_t)z * t.dim[1] + y) * t.dim[0];
        *s = t.cell_start[row + x0];
        *e = t.cell_start[row + x1 + 1];
    };
    return knn_label_27<KT>(rows, t.sorted, cx, cy, cz, t.dim, qx, qy, qz, k, thr);
}

// the same against any target: a target of fewer than k points (s_t, in shared memory) by brute force
__device__ __forceinline__ uint8_t knn_label_dispatch(const KnnTarget& t, const float4* s_t, float qx, float qy, float qz, int k, float thr) {
    if (t.small.n > 0) return knn_label_all<kKnnMaxK>((int)t.small.n, [&](int p) { return s_t[p]; }, qx, qy, qz, k, thr);
    switch (k) {
        case 1: return knn_label<1>(t, qx, qy, qz, k, thr);
        case 2: return knn_label<2>(t, qx, qy, qz, k, thr);
        case 3: return knn_label<3>(t, qx, qy, qz, k, thr);
        case 4: return knn_label<4>(t, qx, qy, qz, k, thr);
        default: return knn_label<kKnnMaxK>(t, qx, qy, qz, k, thr);
    }
}

// a target of fewer than k points (at most kKnnMaxK - 1) into shared memory, for knn_label_dispatch
__device__ __forceinline__ void load_small_target(const KnnTarget& t, float4* s_t) {
    if (t.small.n > 0 && threadIdx.x < t.small.n) s_t[threadIdx.x] = make_float4(t.small.x[threadIdx.x], t.small.y[threadIdx.x], t.small.z[threadIdx.x], 0.0f);
    if (t.small.n > 0) __syncthreads();
}

// scans: local -> (base2lidar as written at Session.cpp:545) -> pose => global query, then, with T16 != null, the points of an accepted
// keyframe moved by its float 4x4 in f32 (Session.cpp:565); label.  sm_90a: 40 registers, no spill, 12 CTAs per SM.  The minimum of 12
// CTAs keeps that allocation: with the bare bound ptxas picks 32 registers and a 44 B spill since the kernel carries the refinement.
__global__ void __launch_bounds__(128, 12) knn_scan_label_kernel(PtrView scans, const int64_t* __restrict__ off, int K, const double* __restrict__ poses,
                                                             const double* __restrict__ ext, int order, const float* __restrict__ T16,
                                                             const uint8_t* __restrict__ accept, KnnTarget t, int k, float thr,
                                                             uint8_t* __restrict__ label, float* __restrict__ gx, float* __restrict__ gy,
                                                             float* __restrict__ gz) {
    __shared__ float4 s_t[kKnnMaxK];
    load_small_target(t, s_t);
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= scans.n) return;
    const int kf = find_kf(off, K, i);
    float x = scans.x[i], y = scans.y[i], z = scans.z[i];
    scan_to_global(poses + (size_t)kf * 24 + 12, ext, order, &x, &y, &z);
    refine_point(T16, accept, kf, &x, &y, &z);
    gx[i] = x; gy[i] = y; gz[i] = z;
    label[i] = knn_label_dispatch(t, s_t, x, y, z, k, thr);
}

// sm_90a: 32 registers and a 44 B spill (L1-resident) at full occupancy, which the minimum of 16 CTAs per SM keeps (the bare bound gives
// 40 registers).  __launch_bounds__(128, 12) removes the spill (40 registers) but was measured 11 % slower on an H100 (4 M queries
// against 1 M targets, k = 2: 0.67 vs 0.61 ms).
__global__ void __launch_bounds__(128, 16) knn_cloud_label_kernel(PtrView q, KnnTarget t, int k, float thr, uint8_t* __restrict__ label) {
    __shared__ float4 s_t[kKnnMaxK];
    load_small_target(t, s_t);
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= q.n) return;
    label[i] = knn_label_dispatch(t, s_t, q.x[i], q.y[i], q.z[i], k, thr);
}

int knn_target_build(ltr_ctx* ctx, const DevCloud& target, int k, float thr, KnnTarget* t, void** block) {
    *t = KnnTarget();
    if (target.n < k) { t->small = view(target); return LTR_OK; }
    float mn[3], mx[3];
    // an infinite or NaN extent would keep the cell loop below from ever terminating.  Targets of the path are voxelised maps,
    // which the voxeliser has already checked, so nothing reproduces PCL's skipping of invalid points here.
    LTR_TRY(finite_extent(ctx, target, "target", mn, mx));
    const double reach = std::sqrt((double)k * (double)thr) * 1.001 + 1e-6;
    double cell = reach;
    // bound the dense grid to 2^29 cells by growing the cell (exactness only needs cell >= reach)
    for (;;) {
        double cells = 1.0;
        for (int d = 0; d < 3; ++d) cells *= std::floor(((double)mx[d] - (double)mn[d]) / cell) + 3.0;
        if (cells <= 536870912.0) break;
        cell *= 1.25;
    }
    KnnTarget g;
    g.inv_cell = 1.0 / cell;
    size_t ncell = 1;
    for (int d = 0; d < 3; ++d) {
        g.origin[d] = (double)mn[d] - cell;  // one guard cell below the minimum
        g.dim[d] = (int)std::floor(((double)mx[d] - g.origin[d]) * g.inv_cell) + 2;
        ncell *= (size_t)g.dim[d];
    }
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);   // handed to the caller (*block) only when the grid is complete
    const size_t cs_bytes = (ncell + 1) * sizeof(uint32_t);
    const size_t cs_pad = (cs_bytes + 255) / 256 * 256;
    LTR_TRY(dev_alloc(ctx, &p, 2 * cs_pad + (size_t)target.n * sizeof(float4)));
    uint32_t* cnt = (uint32_t*)p;
    uint32_t* start = (uint32_t*)((char*)p + cs_pad);
    float4* sorted = (float4*)((char*)p + 2 * cs_pad);
    g.cell_start = start;
    g.sorted = sorted;
    LTR_CUDA(ctx, cudaMemsetAsync(cnt, 0, cs_pad, ctx->stream));
    const unsigned nb = (unsigned)((target.n + 255) / 256);
    grid_count_kernel<<<nb, 256, 0, ctx->stream>>>(view(target), g, cnt);
    LTR_LAUNCH_CHECK(ctx);
    LTR_TRY(exclusive_scan_u32(ctx, cnt, start, (int64_t)ncell + 1));
    LTR_CUDA(ctx, cudaMemsetAsync(cnt, 0, cs_pad, ctx->stream));
    grid_fill_kernel<<<nb, 256, 0, ctx->stream>>>(view(target), g, cnt, sorted);
    LTR_LAUNCH_CHECK(ctx);
    *t = g;
    *block = p;
    p = nullptr;   // ownership moves to the caller
    return LTR_OK;
}

int knn_target_label(ltr_ctx* ctx, const KnnTarget& t, PtrView q, int k, float thr, uint8_t* label) {
    if (q.n == 0) return LTR_OK;
    knn_cloud_label_kernel<<<(unsigned)((q.n + 127) / 128), 128, 0, ctx->stream>>>(q, t, k, thr, label);
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

int knn_diff(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud target_h, int32_t k, float thr, bool refined,
             const float* T16, const uint8_t* accepted, ltr_scanset* out_coexist, ltr_scanset* out_diff) {
    DevScanSet* sp;
    DevPoses* pp;
    DevCloud* tp;
    LTR_TRY(scanset_get(ctx, scans_h, &sp));
    LTR_TRY(poses_get(ctx, poses_h, &pp));
    LTR_TRY(cloud_get(ctx, target_h, &tp));
    if (k < 1 || k > kKnnMaxK) return fail(ctx, LTR_ERR_UNSUPPORTED, "k = %d outside [1, %d]", k, kKnnMaxK);
    if (!(thr > 0.0f)) return fail(ctx, LTR_ERR_INVALID, "threshold must be positive");
    LTR_TRY(check_pose_range(ctx, *sp, *pp, pose_offset));
    if (tp->n < 1) return fail(ctx, LTR_ERR_UNSUPPORTED, "empty target map (PCL's nearestKSearch asserts on an empty tree)");
    const DevScanSet scans = *sp;
    if (refined && scans.K > 0 && (!T16 || !accepted)) return fail(ctx, LTR_ERR_INVALID, "null transforms or accept mask");
    const DevPoses poses = *pp;
    const DevCloud target = *tp;
    const int64_t n = scans.pts.n;
    const int K = scans.K;
    ScanSplit split(ctx, scans, poses.d + (size_t)pose_offset * 24);
    LTR_TRY(split.init());
    if (n > 0) {
        KnnTarget t;
        void* t_block = nullptr;
        ScratchGuard g_grid(ctx, &t_block);
        LTR_TRY(knn_target_build(ctx, target, k, thr, &t, &t_block));
        void* p = nullptr;
        ScratchGuard g_p(ctx, &p);
        const size_t b_g = ((size_t)n * 12 + 255) / 256 * 256, b_T = T16 ? ((size_t)K * 64 + 255) / 256 * 256 : 0;
        LTR_TRY(dev_alloc(ctx, &p, b_g + b_T + (T16 ? (size_t)K : 0)));
        float* gx = (float*)p;
        float* gy = gx + n;
        float* gz = gy + n;
        float* dT = nullptr;
        uint8_t* dacc = nullptr;
        if (T16) {
            dT = (float*)((char*)p + b_g);
            dacc = (uint8_t*)p + b_g + b_T;
            LTR_TRY(upload_refinement(ctx, K, T16, accepted, dT, dacc));
        }
        knn_scan_label_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(view(scans.pts), scans.d_off, K, poses.d + (size_t)pose_offset * 24,
            ctx->ext_identity ? nullptr : ctx->d_ext, ctx->cfg.transform_order, dT, dacc, t, k, thr, split.flags, gx, gy, gz);
        LTR_LAUNCH_CHECK(ctx);
        g_grid.release();
        // every point goes back; partitioning afterwards keeps the arithmetic identical to the reference, which transforms the two
        // partitions separately with the same per-point operations
        LTR_TRY(split.relocalise(0, n, gx, gy, gz));
    }
    return split.finish(out_coexist, out_diff);
}

}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_knn_diff(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud target_h, int32_t k, float thr,
                 ltr_scanset* out_coexist, ltr_scanset* out_diff) {
    ApiTrace tr__(ctx, "ltr_knn_diff");
    if (!ctx) return LTR_ERR_INVALID;
    return knn_diff(ctx, scans_h, poses_h, pose_offset, target_h, k, thr, false, nullptr, nullptr, out_coexist, out_diff);
}

int ltr_knn_split_cloud(ltr_ctx* ctx, ltr_cloud query_h, ltr_cloud target_h, int32_t k, float thr, ltr_cloud* out_near, ltr_cloud* out_far) {
    ApiTrace tr__(ctx, "ltr_knn_split_cloud");
    if (!ctx || !out_near || !out_far) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevCloud *qp, *tp;
    LTR_TRY(cloud_get(ctx, query_h, &qp));
    LTR_TRY(cloud_get(ctx, target_h, &tp));
    if (k < 1 || k > kKnnMaxK) return fail(ctx, LTR_ERR_UNSUPPORTED, "k = %d outside [1, %d]", k, kKnnMaxK);
    if (!(thr > 0.0f)) return fail(ctx, LTR_ERR_INVALID, "threshold must be positive");
    if (tp->n < 1) return fail(ctx, LTR_ERR_UNSUPPORTED, "empty target (PCL's nearestKSearch asserts on an empty tree)");
    const DevCloud q = *qp, target = *tp;
    KnnTarget t;
    void* t_block = nullptr;
    ScratchGuard g_grid(ctx, &t_block);
    if (q.n > 0) LTR_TRY(knn_target_build(ctx, target, k, thr, &t, &t_block));   // before the outputs exist, so that a rejected target leaks nothing
    CloudOwner near_, far_;
    LTR_TRY(cloud_new(ctx, q.n, &near_));
    LTR_TRY(cloud_new(ctx, q.n, &far_));
    if (q.n > 0) {
        void* p = nullptr;
        ScratchGuard g_p(ctx, &p);
        LTR_TRY(dev_alloc(ctx, &p, (size_t)q.n));
        LTR_TRY(knn_target_label(ctx, t, view(q), k, thr, (uint8_t*)p));
        g_grid.release();
        DevCloud o0 = ctx->clouds[near_.get()], o1 = ctx->clouds[far_.get()];
        int64_t nf = 0;
        LTR_TRY(stable_partition_by_flag(ctx, q, (const uint8_t*)p, &nf, &o0, &o1));
        ctx->clouds[near_.get()].n = o0.n;
        ctx->clouds[far_.get()].n = o1.n;
    }
    *out_near = near_.release();
    *out_far = far_.release();
    return LTR_OK;
}

}  // extern "C"
