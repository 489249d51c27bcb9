// libltr_b200.so -- ICP refinement of the low-dynamic kNN diff: every keyframe is registered to the other session's 0.4 m map before the
// change test.
//
// Reference (live code behind a constant, `bool useICPrefinement { false }`):
//   Session::extractLowDynPointsViaKnnDiff        ltremovert/src/Session.cpp:393-427   ICP set-up, 0.4 m target
//   Session::partitionLowDynamicPointsOfScanByKnn ltremovert/src/Session.cpp:549-584   0.4 m source, align, accept iff fitness < 1.0
// PCL's IterativeClosestPoint<PointXYZI, PointXYZI> (float) cannot be reproduced bit for bit: its arithmetic lives in Eigen (umeyama,
// JacobiSVD, packet-order reductions) and FLANN (tie order).  The contract keeps PCL's control flow and the reference's parameters and
// fixes the arithmetic; the device equals the CPU restatement tests/_icp_oracle.py bit for bit (DESIGN.md §5.2).  For keyframe k of the
// scan set (pose index pose_offset + k):
//  1. scan_global = local2global(scan_k, pose, base2lidar) exactly as ltr_knn_diff moves it (the reference's choice of extrinsic);
//     ltr_icp_refine_scanside instead moves it as ltr_scanside_split does, local2global(scan_k, pose, lidar2base) (utility.cpp:160-168,
//     the scan-side registration of Removerter.cpp:950-1017); with the identity extrinsic the two agree bit for bit.
//     src = octreeDownsampling(scan_global, source_leaf) (ltr_voxel_centroid_per_keyframe); tgt = the caller's 0.4 m target.
//  2. Correspondences (CorrespondenceEstimation::determineCorrespondences): the partner of each working source point is its nearest tgt
//     point by L2_Simple in f32 (((dx*dx) + dy*dy) + dz*dz, no FMA), the LOWEST tgt index on ties; pairs with (double)d2 > max_dist^2 are
//     dropped; correspondences are in source order.
//  3. Rigid estimate: means and the 3x3 cross-covariance H = sum (p - p_mean)(q - q_mean)^T in double from the f32 coordinates; the
//     rotation is Horn's unit quaternion, the eigenvector of the largest eigenvalue (lowest index on ties) of his symmetric 4x4 matrix N(H),
//     found by kJacobiSweeps cyclic Jacobi sweeps over the pairs (0,1) (0,2) (0,3) (1,2) (1,3) (2,3).  Horn's maximum is taken over proper
//     rotations only, i.e. it is the SVD solution with the reflection fix det(V U^T) < 0 -> flip.  t = q_mean - R p_mean; R and t are
//     rounded once to a float 4x4 (PCL's Matrix4f).
//     Reduction shape (every sum of the loop and of the fitness): thread j of the keyframe's CTA (kIcpThreads = B threads) adds the terms
//     of points j, j + B, j + 2B, ... sequentially in double from 0.0; then a binary tree over the B partials, stride B/2 down to 1,
//     partial[j] = partial[j] + partial[j + stride].  No floating-point atomics.
//  4. Iteration (IterativeClosestPoint::computeTransformation): fewer than min_correspondences correspondences -> exit 5, stop.  Else
//     estimate T_inc, move the working source by it in f32 as ((m0 x + m1 y) + m2 z) + m3, compose final = T_inc final as an f32 4x4
//     product summed ((T[r][0] F[0][c] + T[r][1] F[1][c]) + T[r][2] F[2][c]) + T[r][3] F[3][c], ++iterations.
//  5. Convergence (DefaultConvergenceCriteria, max_iterations_similar_transforms_ = 0), in this order:
//     1 iterations >= max_iterations; 2 0.5 * (double)(((T00 + T11) + T22) - 1.0f) >= 1 - transformation_epsilon and
//     (double)((tx*tx + ty*ty) + tz*tz) <= transformation_epsilon (float sums, as PCL's float coefficients promote); 3 |mse - prev_mse|
//     < mse_threshold_absolute; 4 |mse - prev_mse| / prev_mse < euclidean_fitness_epsilon.  mse = (sum of this iteration's correspondence
//     d2) / count, prev_mse starts at DBL_MAX.
//  6. Fitness (getFitnessScore(DBL_MAX)): src (the ORIGINAL 0.4 m source) moved by final in f32, mean of the nearest d2 to tgt in double;
//     no points -> DBL_MAX.
// The partition (ltr_knn_diff_refined) then moves scan_global by final in f32 when the caller accepts the keyframe (the reference: fitness
// < 1.0) and runs ltr_knn_diff's labelling and global2local on it, so a keyframe that is not accepted gives ltr_knn_diff's bytes.
//
// Nearest neighbour with index.  tgt goes into the sparse grid levels of sparse_grid.cuh (one segment, built once per call: the target is
// fixed across iterations).  A query searches shell by shell; on a level it stops after shell s >= 1 when its current smallest distance D
// satisfies D <= ((s - 2^-6) c)^2 (1 - 2^-20), or when the block holds every cell, but not at D = 0 in shell 0.  sparse_grid.cuh's header
// proves that the lowest index among the points at distance D is then the lowest overall.  Bounded levels give up after kNnShells
// shells and the query moves to the next, 4x coarser level; the coarsest searches until the rule holds.
//
// Memory: the global scans (16 B/point) while the source is voxelised, the 0.4 m source (16 B per source point), tgt's grid levels (28 B
// per tgt point each), and per launch of at most LTR_ICP_CHUNK_POINTS source points (environment; default 2^24, a keyframe is never
// split) a working copy and a correspondence index (20 B per source point).  All of it comes from the context's allocator and is
// returned before the call ends.
#include "ltr_internal.cuh"
#include "ref_math.cuh"
#include "sparse_grid.cuh"
#include <algorithm>
#include <cfloat>
#include <cmath>

namespace ltr {

namespace {

constexpr int kIcpThreads = 256;      // B of the reduction shape
constexpr int kJacobiSweeps = 10;
constexpr int kNnShells = 2;
constexpr int64_t kChunkPoints = (int64_t)1 << 24;
constexpr int kExitNoCorrespondences = LTR_ICP_NO_CORRESPONDENCES;

struct Levels {
    Level L[kGridMaxLevels];
    int n;
};

struct IcpArgs {
    double max_d2, rot_thr, trans_thr, mse_abs, mse_rel;
    int max_it, min_corr;
};

LTR_DEV double ds(double a, double b) { return __dsub_rn(a, b); }
LTR_DEV double dd(double a, double b) { return __ddiv_rn(a, b); }

// ---- exact 1-NN with the lowest index on ties (file header) --------------------------------------------------------------------------
// the shell search's accumulator; its stop rule is in sparse_grid.cuh's header
struct Nearest {
    float d;
    uint32_t i;
    LTR_DEV void push(float v, const float4& t) {
        const uint32_t idx = __float_as_uint(t.w);
        if (v < d || (v == d && idx < i)) { d = v; i = idx; }
    }
    LTR_DEV bool settled(long long s, double cell) const { return i != 0xffffffffu && s > 0 && (double)d <= shell_bound(s, cell); }
};

LTR_DEV void nn1(const Levels& T, float qx, float qy, float qz, float* d, uint32_t* idx) {
    for (int l = 0; l < T.n; ++l) {
        Nearest b{__int_as_float(0x7f800000), 0xffffffffu};
        if (shell_search(T.L[l], 0, qx, qy, qz, kNnShells, b)) { *d = b.d; *idx = b.i; return; }
    }
}

// ---- rigid estimate (file header, step 3) -------------------------------------------------------------------------------------------
// H[3a + b] = sum (p_a - p_mean_a)(q_b - q_mean_b); writes R (row-major 3x3) and t in double.
LTR_DEV void horn_rigid(const double* H, const double* pm, const double* qm, double* R, double* t) {
    const double Sxx = H[0], Sxy = H[1], Sxz = H[2], Syx = H[3], Syy = H[4], Syz = H[5], Szx = H[6], Szy = H[7], Szz = H[8];
    double A[4][4];
    A[0][0] = da(da(Sxx, Syy), Szz);
    A[1][1] = ds(ds(Sxx, Syy), Szz);
    A[2][2] = ds(da(-Sxx, Syy), Szz);
    A[3][3] = da(ds(-Sxx, Syy), Szz);
    A[0][1] = A[1][0] = ds(Syz, Szy);
    A[0][2] = A[2][0] = ds(Szx, Sxz);
    A[0][3] = A[3][0] = ds(Sxy, Syx);
    A[1][2] = A[2][1] = da(Sxy, Syx);
    A[1][3] = A[3][1] = da(Szx, Sxz);
    A[2][3] = A[3][2] = da(Syz, Szy);
    double V[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) V[r][c] = r == c ? 1.0 : 0.0;
    const int P[6] = {0, 0, 0, 1, 1, 2}, Q[6] = {1, 2, 3, 2, 3, 3};
#pragma unroll 1
    for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            const int p = P[j], q = Q[j];
            const double apq = A[p][q];
            if (apq == 0.0) continue;
            const double theta = dd(ds(A[q][q], A[p][p]), dm(2.0, apq));
            double tt = dd(1.0, da(fabs(theta), __dsqrt_rn(da(dm(theta, theta), 1.0))));
            if (theta < 0.0) tt = -tt;
            const double c = dd(1.0, __dsqrt_rn(da(dm(tt, tt), 1.0))), s = dm(tt, c);
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                if (r == p || r == q) continue;
                const double arp = A[r][p], arq = A[r][q];
                A[r][p] = A[p][r] = ds(dm(c, arp), dm(s, arq));
                A[r][q] = A[q][r] = da(dm(s, arp), dm(c, arq));
            }
            const double app = A[p][p], aqq = A[q][q];
            A[p][p] = ds(app, dm(tt, apq));
            A[q][q] = da(aqq, dm(tt, apq));
            A[p][q] = A[q][p] = 0.0;
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const double vrp = V[r][p], vrq = V[r][q];
                V[r][p] = ds(dm(c, vrp), dm(s, vrq));
                V[r][q] = da(dm(s, vrp), dm(c, vrq));
            }
        }
    }
    int m = 0;
#pragma unroll
    for (int j = 1; j < 4; ++j) if (A[j][j] > A[m][m]) m = j;
    double w = V[0][m], x = V[1][m], y = V[2][m], z = V[3][m];
    const double nrm = __dsqrt_rn(da(da(da(dm(w, w), dm(x, x)), dm(y, y)), dm(z, z)));
    w = dd(w, nrm); x = dd(x, nrm); y = dd(y, nrm); z = dd(z, nrm);
    const double ww = dm(w, w), xx = dm(x, x), yy = dm(y, y), zz = dm(z, z);
    const double wx = dm(w, x), wy = dm(w, y), wz = dm(w, z), xy = dm(x, y), xz = dm(x, z), yz = dm(y, z);
    R[0] = ds(ds(da(ww, xx), yy), zz);
    R[1] = dm(2.0, ds(xy, wz));
    R[2] = dm(2.0, da(xz, wy));
    R[3] = dm(2.0, da(xy, wz));
    R[4] = ds(da(ds(ww, xx), yy), zz);
    R[5] = dm(2.0, ds(yz, wx));
    R[6] = dm(2.0, ds(xz, wy));
    R[7] = dm(2.0, da(yz, wx));
    R[8] = da(ds(ds(ww, xx), yy), zz);
#pragma unroll
    for (int a = 0; a < 3; ++a) t[a] = ds(qm[a], da(da(dm(R[3 * a], pm[0]), dm(R[3 * a + 1], pm[1])), dm(R[3 * a + 2], pm[2])));
}

// binary tree over the B partials of nq sums (file header); the caller has written red[q][tid] and synchronised nothing yet
LTR_DEV void block_tree(double (*red)[kIcpThreads], int nq) {
    __syncthreads();
#pragma unroll 1
    for (int stride = kIcpThreads / 2; stride > 0; stride >>= 1) {
        if ((int)threadIdx.x < stride)
            for (int q = 0; q < nq; ++q) red[q][threadIdx.x] = da(red[q][threadIdx.x], red[q][threadIdx.x + stride]);
        __syncthreads();
    }
}

// One CTA per keyframe kf0 + blockIdx.x: the whole ICP loop and the fitness pass (file header, steps 2-6).
__global__ void __launch_bounds__(kIcpThreads) icp_kernel(Levels T, PtrView tgt, PtrView src, const int64_t* __restrict__ src_off, int kf0,
                                                          int64_t base, IcpArgs a, float4* __restrict__ work, int32_t* __restrict__ corr,
                                                          float* __restrict__ T16, double* __restrict__ fitness, int32_t* __restrict__ iters,
                                                          int32_t* __restrict__ exits) {
    __shared__ double red[9][kIcpThreads];
    __shared__ double s_mean[6], s_mse;
    __shared__ float s_T[16], s_F[16];
    __shared__ int s_cnt, s_stop;
    const int kf = kf0 + blockIdx.x, tid = threadIdx.x;
    const int64_t b = src_off[kf], n = src_off[kf + 1] - b;
    float4* w = work + (b - base);
    int32_t* cr = corr + (b - base);
    for (int64_t i = tid; i < n; i += kIcpThreads) w[i] = make_float4(src.x[b + i], src.y[b + i], src.z[b + i], 0.0f);
    double prev_mse = DBL_MAX;   // thread 0's convergence state
    int it = 0, ex = 0;
    if (tid == 0) {
        for (int j = 0; j < 16; ++j) s_F[j] = (j % 5 == 0) ? 1.0f : 0.0f;
        s_stop = 0;
    }
    for (;;) {
        if (tid == 0) s_cnt = 0;
        __syncthreads();
        // correspondences and their first sums
        int cnt = 0;
        double acc[7] = {0, 0, 0, 0, 0, 0, 0};
        for (int64_t i = tid; i < n; i += kIcpThreads) {
            const float4 p = w[i];
            float d;
            uint32_t j;
            nn1(T, p.x, p.y, p.z, &d, &j);
            if ((double)d <= a.max_d2) {
                cr[i] = (int32_t)j;
                ++cnt;
                acc[0] = da(acc[0], (double)p.x); acc[1] = da(acc[1], (double)p.y); acc[2] = da(acc[2], (double)p.z);
                acc[3] = da(acc[3], (double)tgt.x[j]); acc[4] = da(acc[4], (double)tgt.y[j]); acc[5] = da(acc[5], (double)tgt.z[j]);
                acc[6] = da(acc[6], (double)d);
            } else {
                cr[i] = -1;
            }
        }
        if (cnt) atomicAdd(&s_cnt, cnt);
        for (int q = 0; q < 7; ++q) red[q][tid] = acc[q];
        block_tree(red, 7);
        if (tid == 0) {
            if (s_cnt < a.min_corr) { ex = kExitNoCorrespondences; s_stop = 1; }
            else {
                const double c = (double)s_cnt;
                for (int q = 0; q < 6; ++q) s_mean[q] = dd(red[q][0], c);
                s_mse = dd(red[6][0], c);
            }
        }
        __syncthreads();
        if (s_stop) break;
        // cross-covariance
        double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
        const double pm[3] = {s_mean[0], s_mean[1], s_mean[2]}, qm[3] = {s_mean[3], s_mean[4], s_mean[5]};
        for (int64_t i = tid; i < n; i += kIcpThreads) {
            const int32_t j = cr[i];
            if (j < 0) continue;
            const float4 p = w[i];
            const double dp[3] = {ds((double)p.x, pm[0]), ds((double)p.y, pm[1]), ds((double)p.z, pm[2])};
            const double dq[3] = {ds((double)tgt.x[j], qm[0]), ds((double)tgt.y[j], qm[1]), ds((double)tgt.z[j], qm[2])};
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) h[3 * r + c] = da(h[3 * r + c], dm(dp[r], dq[c]));
        }
        for (int q = 0; q < 9; ++q) red[q][tid] = h[q];
        block_tree(red, 9);
        if (tid == 0) {
            double H[9], R[9], t[3];
            for (int q = 0; q < 9; ++q) H[q] = red[q][0];
            horn_rigid(H, pm, qm, R, t);
            for (int r = 0; r < 3; ++r) {
                for (int c = 0; c < 3; ++c) s_T[4 * r + c] = __double2float_rn(R[3 * r + c]);
                s_T[4 * r + 3] = __double2float_rn(t[r]);
            }
            s_T[12] = 0.0f; s_T[13] = 0.0f; s_T[14] = 0.0f; s_T[15] = 1.0f;
            float F[16];
            for (int r = 0; r < 4; ++r)
                for (int c = 0; c < 4; ++c)
                    F[4 * r + c] = fa(fa(fa(fm(s_T[4 * r], s_F[c]), fm(s_T[4 * r + 1], s_F[4 + c])), fm(s_T[4 * r + 2], s_F[8 + c])),
                                      fm(s_T[4 * r + 3], s_F[12 + c]));
            for (int j = 0; j < 16; ++j) s_F[j] = F[j];
            ++it;
            const double cos_angle = dm(0.5, (double)fs(fa(fa(s_T[0], s_T[5]), s_T[10]), 1.0f));
            const double tsq = (double)fa(fa(fm(s_T[3], s_T[3]), fm(s_T[7], s_T[7])), fm(s_T[11], s_T[11]));
            const double mse = s_mse, dmse = fabs(ds(mse, prev_mse));
            if (it >= a.max_it) ex = LTR_ICP_ITERATIONS;
            else if (cos_angle >= a.rot_thr && tsq <= a.trans_thr) ex = LTR_ICP_TRANSFORM;
            else if (dmse < a.mse_abs) ex = LTR_ICP_ABS_MSE;
            else if (dd(dmse, prev_mse) < a.mse_rel) ex = LTR_ICP_REL_MSE;
            prev_mse = mse;
            s_stop = ex != 0;
        }
        __syncthreads();
        for (int64_t i = tid; i < n; i += kIcpThreads) {
            const float4 p = w[i];
            w[i] = make_float4(frow(s_T, p.x, p.y, p.z), frow(s_T + 4, p.x, p.y, p.z), frow(s_T + 8, p.x, p.y, p.z), 0.0f);
        }
        if (s_stop) break;
    }
    __syncthreads();
    // fitness: the original source moved by final
    double fs_sum = 0.0;
    int fc = 0;
    for (int64_t i = tid; i < n; i += kIcpThreads) {
        const float x = src.x[b + i], y = src.y[b + i], z = src.z[b + i];
        float d;
        uint32_t j;
        nn1(T, frow(s_F, x, y, z), frow(s_F + 4, x, y, z), frow(s_F + 8, x, y, z), &d, &j);
        if ((double)d <= DBL_MAX) { fs_sum = da(fs_sum, (double)d); ++fc; }
    }
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    if (fc) atomicAdd(&s_cnt, fc);
    red[0][tid] = fs_sum;
    block_tree(red, 1);
    if (tid == 0) {
        fitness[kf] = s_cnt > 0 ? dd(red[0][0], (double)s_cnt) : DBL_MAX;
        iters[kf] = it;
        exits[kf] = ex;
        for (int j = 0; j < 16; ++j) T16[16 * (size_t)kf + j] = s_F[j];
    }
}

// every level of pyr up to the final one: nn1 may search all of them
int build_all_levels(Pyramid& pyr, Levels* lv) {
    *lv = Levels{};
    for (int l = 0;; ++l) {
        const Level* L;
        LTR_TRY(pyr.get(l, &L));
        lv->L[l] = *L;
        lv->n = l + 1;
        if (L->final_level) return LTR_OK;
    }
}

__global__ void __launch_bounds__(256) nearest_debug_kernel(Levels T, PtrView q, float* __restrict__ d, int32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= q.n) return;
    float v;
    uint32_t j;
    nn1(T, q.x[i], q.y[i], q.z[i], &v, &j);
    d[i] = v;
    idx[i] = (int32_t)j;
}

}  // namespace
}  // namespace ltr

using namespace ltr;

extern "C" void ltr_icp_params_default(ltr_icp_params* p) {
    if (!p) return;
    p->max_correspondence_distance = 150.0;   // Session.cpp:396
    p->max_iterations = 100;                  // :397
    p->transformation_epsilon = 1e-6;         // :398
    p->euclidean_fitness_epsilon = 1e-6;      // :399
    p->mse_threshold_absolute = 1e-12;        // DefaultConvergenceCriteria's default
    p->min_correspondences = 3;               // IterativeClosestPoint's default
    p->source_leaf = 0.4f;                    // Session.cpp:558-559
}

namespace ltr {
namespace {

// ltr_icp_refine (scanside = false: scan_global as ltr_knn_diff moves it, base2lidar then the pose) and ltr_icp_refine_scanside
// (scanside = true: as ltr_scanside_split moves it, lidar2base then the pose); everything after step 1 is the same.
int icp_refine(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud target_h, const ltr_icp_params* prm,
               bool scanside, float* T16_out, double* fitness_out, int32_t* iterations_out, int32_t* exit_out) {
    ltr_icp_params P;
    ltr_icp_params_default(&P);
    if (prm) P = *prm;
    if (!(P.max_correspondence_distance > 0.0) || P.max_iterations < 1 || !(P.transformation_epsilon >= 0.0) ||
        !(P.euclidean_fitness_epsilon >= 0.0) || !(P.mse_threshold_absolute >= 0.0) || P.min_correspondences < 1 ||
        !(P.source_leaf > 0.0f) || !std::isfinite(P.source_leaf))
        return fail(ctx, LTR_ERR_INVALID, "invalid ICP parameters");
    DevScanSet* sp;
    DevPoses* pp;
    DevCloud* tp;
    LTR_TRY(scanset_get(ctx, scans_h, &sp));
    LTR_TRY(poses_get(ctx, poses_h, &pp));
    LTR_TRY(check_pose_range(ctx, *sp, *pp, pose_offset));
    LTR_TRY(cloud_get(ctx, target_h, &tp));
    if (tp->n < 1) return fail(ctx, LTR_ERR_UNSUPPORTED, "empty ICP target");
    const DevScanSet scans = *sp;
    const DevPoses poses = *pp;
    const DevCloud tgt = *tp;
    const int K = scans.K;
    float tmn[3], tmx[3];
    LTR_TRY(finite_extent(ctx, tgt, "ICP target", tmn, tmx));
    std::vector<float> hT((size_t)K * 16);
    std::vector<double> hfit((size_t)K, DBL_MAX);
    std::vector<int32_t> hit((size_t)K, 0), hex((size_t)K, kExitNoCorrespondences);
    for (int k = 0; k < K; ++k)
        for (int j = 0; j < 16; ++j) hT[16 * (size_t)k + j] = (j % 5 == 0) ? 1.0f : 0.0f;
    if (scans.pts.n > 0) {
        // 1. the global scans and their per-keyframe 0.4 m centroids
        ScanSetOwner g_glob;
        LTR_TRY(scanset_new(ctx, scans.h_off, &g_glob));
        const DevCloud g = ctx->scansets[g_glob.get()].pts;
        // scan_global as the partition that follows moves it: base2lidar (kNN diff) or lidar2base (scan-side removal), then the pose
        const double* ext = ctx->ext_identity ? nullptr : ctx->d_ext + (scanside ? 12 : 0);
        LTR_TRY(scans_to_global(ctx, scans, 0, scans.pts.n, poses.d + (size_t)pose_offset * 24, ext, g.x(), g.y(), g.z(), g.i()));
        {
            float mn[3], mx[3];
            LTR_TRY(finite_extent(ctx, g, "scan", mn, mx));
        }
        ltr_scanset h_src;
        LTR_TRY(ltr_voxel_centroid_per_keyframe(ctx, g_glob.get(), P.source_leaf, &h_src));
        ScanSetOwner g_src(ctx, h_src);
        g_glob.reset();
        const DevScanSet src = ctx->scansets[g_src.get()];
        // 2. the target's grid levels, all of them: every iteration searches them
        Pyramid pyr(ctx);
        pyr.init(view(tgt), nullptr, 1, tmn, tmx);
        Levels lv;
        LTR_TRY(build_all_levels(pyr, &lv));
        // 3. keyframe chunks of at most LTR_ICP_CHUNK_POINTS source points, one CTA per keyframe
        int64_t max_chunk = 0;
        const std::vector<int> kf_cut = plan_keyframe_chunks(src.h_off, env_points("LTR_ICP_CHUNK_POINTS", kChunkPoints, (int64_t)1 << 30), K,
                                                             &max_chunk);
        if (max_chunk >= ((int64_t)1 << 31)) return fail(ctx, LTR_ERR_UNSUPPORTED, "a keyframe of %lld source points", (long long)max_chunk);
        auto pad = [](size_t v) { return (v + 255) / 256 * 256; };
        const size_t b_work = pad((size_t)std::max<int64_t>(max_chunk, 1) * 16), b_corr = pad((size_t)std::max<int64_t>(max_chunk, 1) * 4);
        const size_t b_T = pad((size_t)K * 64), b_fit = pad((size_t)K * 8), b_i = pad((size_t)K * 4);
        void* blk = nullptr;
        ScratchGuard g_blk(ctx, &blk);
        LTR_TRY(dev_alloc(ctx, &blk, b_work + b_corr + b_T + b_fit + 2 * b_i));
        char* c = (char*)blk;
        float4* work = (float4*)c;
        int32_t* corr = (int32_t*)(c + b_work);
        float* dT = (float*)(c + b_work + b_corr);
        double* dfit = (double*)(c + b_work + b_corr + b_T);
        int32_t* dit = (int32_t*)(c + b_work + b_corr + b_T + b_fit);
        int32_t* dex = (int32_t*)(c + b_work + b_corr + b_T + b_fit + b_i);
        IcpArgs a;
        a.max_d2 = P.max_correspondence_distance * P.max_correspondence_distance;
        a.rot_thr = 1.0 - P.transformation_epsilon;
        a.trans_thr = P.transformation_epsilon;
        a.mse_abs = P.mse_threshold_absolute;
        a.mse_rel = P.euclidean_fitness_epsilon;
        a.max_it = P.max_iterations;
        a.min_corr = P.min_correspondences;
        for (size_t ci = 0; ci + 1 < kf_cut.size(); ++ci) {
            const int kf0 = kf_cut[ci], nkf = kf_cut[ci + 1] - kf0;
            icp_kernel<<<nkf, kIcpThreads, 0, ctx->stream>>>(lv, view(tgt), view(src.pts), src.d_off, kf0, src.h_off[kf0], a, work, corr, dT, dfit,
                                                             dit, dex);
            LTR_LAUNCH_CHECK(ctx);
        }
        LTR_CUDA(ctx, cudaMemcpyAsync(hT.data(), dT, (size_t)K * 64, cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaMemcpyAsync(hfit.data(), dfit, (size_t)K * 8, cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaMemcpyAsync(hit.data(), dit, (size_t)K * 4, cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaMemcpyAsync(hex.data(), dex, (size_t)K * 4, cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (T16_out) std::copy(hT.begin(), hT.end(), T16_out);
    if (fitness_out) std::copy(hfit.begin(), hfit.end(), fitness_out);
    if (iterations_out) std::copy(hit.begin(), hit.end(), iterations_out);
    if (exit_out) std::copy(hex.begin(), hex.end(), exit_out);
    return LTR_OK;
}

}  // namespace
}  // namespace ltr

extern "C" {

int ltr_icp_refine(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud target_h, const ltr_icp_params* prm,
                   float* T16_out, double* fitness_out, int32_t* iterations_out, int32_t* exit_out) {
    ApiTrace tr__(ctx, "ltr_icp_refine");
    if (!ctx) return LTR_ERR_INVALID;
    return icp_refine(ctx, scans_h, poses_h, pose_offset, target_h, prm, false, T16_out, fitness_out, iterations_out, exit_out);
}

int ltr_icp_refine_scanside(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud target_h,
                            const ltr_icp_params* prm, float* T16_out, double* fitness_out, int32_t* iterations_out, int32_t* exit_out) {
    ApiTrace tr__(ctx, "ltr_icp_refine_scanside");
    if (!ctx) return LTR_ERR_INVALID;
    return icp_refine(ctx, scans_h, poses_h, pose_offset, target_h, prm, true, T16_out, fitness_out, iterations_out, exit_out);
}

int ltr_knn_diff_refined(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud target_h, int32_t k, float thr,
                         const float* T16, const uint8_t* accepted, ltr_scanset* out_coexist, ltr_scanset* out_diff) {
    ApiTrace tr__(ctx, "ltr_knn_diff_refined");
    if (!ctx) return LTR_ERR_INVALID;
    DevScanSet* sp;
    DevPoses* pp;
    LTR_TRY(scanset_get(ctx, scans_h, &sp));
    LTR_TRY(poses_get(ctx, poses_h, &pp));
    LTR_TRY(check_pose_range(ctx, *sp, *pp, pose_offset));   // this entry checks the pose range before k and thr
    return knn_diff(ctx, scans_h, poses_h, pose_offset, target_h, k, thr, true, T16, accepted, out_coexist, out_diff);
}

// The correspondence search of ltr_icp_refine (nn1 over every level of the target's pyramid) for every point of query_h.
int ltr_debug_nearest(ltr_ctx* ctx, ltr_cloud query_h, ltr_cloud target_h, float* d_out, int32_t* idx_out) {
    ApiTrace tr__(ctx, "ltr_debug_nearest");
    if (!ctx || !d_out || !idx_out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevCloud* qp;
    DevCloud* tp;
    LTR_TRY(cloud_get(ctx, query_h, &qp));
    LTR_TRY(cloud_get(ctx, target_h, &tp));
    if (tp->n < 1) return fail(ctx, LTR_ERR_UNSUPPORTED, "empty target");
    const DevCloud q = *qp, tgt = *tp;
    float mn[3], mx[3];
    if (q.n > 0) LTR_TRY(finite_extent(ctx, q, "query", mn, mx));
    LTR_TRY(finite_extent(ctx, tgt, "target", mn, mx));
    if (q.n == 0) return LTR_OK;
    Pyramid pyr(ctx);
    pyr.init(view(tgt), nullptr, 1, mn, mx);
    Levels lv;
    LTR_TRY(build_all_levels(pyr, &lv));
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, (size_t)q.n * 8));
    float* dd = (float*)p;
    int32_t* di = (int32_t*)(dd + q.n);
    nearest_debug_kernel<<<(unsigned)((q.n + 255) / 256), 256, 0, ctx->stream>>>(lv, view(q), dd, di);
    LTR_LAUNCH_CHECK(ctx);
    LTR_CUDA(ctx, cudaMemcpyAsync(d_out, dd, (size_t)q.n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaMemcpyAsync(idx_out, di, (size_t)q.n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}

}  // extern "C"
