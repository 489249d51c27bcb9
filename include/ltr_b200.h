/*
 * ltr_b200.h -- C-ABI of the H100-native LT-removert / LT-map hot path (libltr_b200.so).
 *
 * gisbi-kim/lt-mapper exposes no plugin/FFI interface: its surface is the `removert_removert` ROS node
 * and, inside it, the Removerter::run() call graph (ltremovert/src/Removerter.cpp:1653-1678).  This ABI
 * is cut at the narrowest data-parallel seam of that call graph -- the per-keyframe loops and the
 * voxeliser -- so that a host program (ROS/PCL types at its own boundary) keeps the reference's
 * orchestration and calls these entry points where the reference calls the functions cited below.
 * Plain pointers and sizes only; no exceptions cross the boundary; every call returns LTR_OK (0) or
 * a negative ltr_status, with a message retrievable via ltr_last_error().  There is NO CPU fallback:
 * every entry point fails with LTR_ERR_CUDA if no sm_90 device is usable.
 *
 * Conventions
 *  - Points cross the boundary as AoS float[n][4] = x, y, z, intensity (pcl::PointXYZI payload,
 *    ltremovert/include/removert/utility.h:90).  On the device they live as SoA.
 *  - Poses are row-major 4x4 doubles (ltremovert/src/Session.cpp:102-114).  Inverse poses are an INPUT
 *    (the reference computes them with Eigen::Matrix4d::inverse(), Session.cpp:110) so that every
 *    implementation shares the same doubles.
 *  - Handles are small non-negative ints owned by the context; a context is used by one host thread
 *    at a time and is bound to one GPU.
 *  - "cloud"   = one flat device point cloud (a map or any merged cloud),
 *    "scanset" = K per-keyframe clouds stored back to back with K+1 offsets,
 *    "poses"   = K (pose, inverse pose) pairs.
 */
#ifndef LTR_B200_H_
#define LTR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ltr_ctx ltr_ctx;
typedef int32_t ltr_cloud;
typedef int32_t ltr_scanset;
typedef int32_t ltr_poses;

typedef enum ltr_status {
    LTR_OK = 0,
    LTR_ERR_INVALID = -1,      /* bad argument / handle / size (e.g. pose-count != scan-count, Session.cpp:117) */
    LTR_ERR_CUDA = -2,         /* CUDA runtime failure or no usable sm_90 device */
    LTR_ERR_UNSUPPORTED = -3,  /* input the reference itself has undefined behaviour on (e.g. 1- or 2-point maps,
                                  utility.h:158-167 linspace) or outside this build's limits */
    LTR_ERR_NOMEM = -4
} ltr_status;

/* ltr_remove_pass modes == the three variants of calcDescrepancyAndParseDynamicPointIdxForEachScan */
typedef enum ltr_pass_mode {
    LTR_MODE_HD = 0,  /* scan - map  (Removerter.cpp:542-593; removeOnce / revertOnce) */
    LTR_MODE_ND = 1,  /* map - scan  (Removerter.cpp:485-540; iremoveOnceForND)        */
    LTR_MODE_PD = 2   /* scan - map  (Removerter.cpp:429-482; removeOnceForPD)         */
} ltr_pass_mode;

typedef struct ltr_config {
    int32_t device;               /* CUDA device ordinal */
    float vfov_deg, hfov_deg;     /* removert/sequence_vfov, sequence_hfov (RosParamServer.cpp:15-17) */
    double lidar2base[16];        /* kSE3MatExtrinsicLiDARtoPoseBase (RosParamServer.cpp:28-29), row-major */
    double base2lidar[16];        /* its inverse (RosParamServer.cpp:30), supplied by the caller */
    int32_t transform_order;      /* double summation order of pcl::transformPointCloud:
                                     0 = ((m00 x + m01 y) + m02 z) + m03 (PCL <= 1.9), 1 = ((m03 + m00 x) + m01 y) + m02 z (PCL >= 1.10 SSE2) */
    int32_t keyframe_batch;       /* keyframes projected per kernel launch (0 = default) */
    int32_t fast_path;            /* 0 = reference arithmetic for every (point, keyframe) pair; 1 = exactness-preserving fast rejection path;
                                     2 = 1 + tile-level occlusion/range culling for the scan-minus-map variants (default).
                                     With 1 or 2, ltr_parse_projected claims map tiles near to far from each launch's keyframes
                                     (fewer running-minimum atomics; the result does not depend on the order). */
} ltr_config;

/* Fills cfg with the reference defaults (vfov 50, hfov 360, identity extrinsic, order 0). */
void ltr_config_default(ltr_config* cfg);

int ltr_create(ltr_ctx** out, const ltr_config* cfg);
void ltr_destroy(ltr_ctx* ctx);
const char* ltr_last_error(const ltr_ctx* ctx);  /* valid until the next call on ctx; ctx may be NULL for create errors */
int ltr_synchronize(ltr_ctx* ctx);
/* number of kernels of this library launched on ctx so far (for bench.py's gpu_launches) */
int64_t ltr_kernel_launches(const ltr_ctx* ctx);
/* introspection: how many ltr_voxel_centroid* calls found their input already one point per voxel in octree order and skipped the sort */
int64_t ltr_voxel_shortcuts(const ltr_ctx* ctx);
/* introspection: bytes of device memory currently handed out by the context's caching allocator (clouds, scan sets, poses and scratch),
 * bytes parked in its cache, and the high-water mark of the former.  stats3 = { live, cached, peak_live }. */
int ltr_memory_stats(const ltr_ctx* ctx, int64_t* stats3);

/* ---- data movement -------------------------------------------------------------------------- */
/* Page-locked host staging memory for the uploads / downloads below (cudaMallocHost): copies from pageable memory run at a fraction
 * of the link rate and block the caller. */
int ltr_pinned_alloc(size_t bytes, void** out);
void ltr_pinned_free(void* p);
int ltr_cloud_upload(ltr_ctx* ctx, const float* xyzi, int64_t n, ltr_cloud* out);
int ltr_cloud_size(ltr_ctx* ctx, ltr_cloud c, int64_t* n);
int ltr_cloud_download(ltr_ctx* ctx, ltr_cloud c, float* xyzi, int64_t capacity, int64_t* n);
int ltr_cloud_free(ltr_ctx* ctx, ltr_cloud c);
int ltr_cloud_copy(ltr_ctx* ctx, ltr_cloud src, ltr_cloud* out);               /* "*dst = *src" on pcl clouds */
int ltr_cloud_concat(ltr_ctx* ctx, ltr_cloud a, ltr_cloud b, ltr_cloud* out);  /* "*a += *b" result (Removerter.cpp:902 etc.) */
/* Non-owning view of the points [begin, end) of `src` (valid while `src` lives; free it like any cloud, nothing is released).  Lets every rank
 * contribute "its" part of a replicated cloud to ltr_nccl_voxel_centroid_merged. */
int ltr_cloud_slice(ltr_ctx* ctx, ltr_cloud src, int64_t begin, int64_t end, ltr_cloud* out);
/* Device pointers of the SoA components (x, y, z, intensity), e.g. for a caller-side collective. */
int ltr_cloud_device_ptrs(ltr_ctx* ctx, ltr_cloud c, float** x, float** y, float** z, float** i, int64_t* n);
/* Allocates an uninitialised cloud of n points (to be filled through ltr_cloud_device_ptrs). */
int ltr_cloud_alloc(ltr_ctx* ctx, int64_t n, ltr_cloud* out);

int ltr_scanset_upload(ltr_ctx* ctx, const float* xyzi, const int64_t* offsets /* K+1 */, int32_t K, ltr_scanset* out);
int ltr_scanset_info(ltr_ctx* ctx, ltr_scanset s, int32_t* K, int64_t* total_points);
int ltr_scanset_download(ltr_ctx* ctx, ltr_scanset s, float* xyzi, int64_t capacity, int64_t* offsets /* K+1 */);
int ltr_scanset_free(ltr_ctx* ctx, ltr_scanset s);
/* Concatenates the clouds of two scansets keyframe by keyframe: out[k] = a[k] ++ b[k] (Session.cpp:370-371). */
int ltr_scanset_concat_per_keyframe(ltr_ctx* ctx, ltr_scanset a, ltr_scanset b, ltr_scanset* out);
/* View of all points of a scanset as one flat cloud (copy). */
int ltr_scanset_flatten(ltr_ctx* ctx, ltr_scanset s, ltr_cloud* out);

int ltr_poses_upload(ltr_ctx* ctx, const double* poses /* K*16 */, const double* inv_poses /* K*16 */, int32_t K, ltr_poses* out);
int ltr_poses_free(ltr_ctx* ctx, ltr_poses p);

/* ---- hot path ------------------------------------------------------------------------------- */

/* precleaningKeyframes (Session.cpp:506-533): drops points with range < radius and |z| < 0.5. */
int ltr_preclean(ltr_ctx* ctx, ltr_scanset scans, float radius, ltr_scanset* out);

/* mergeScansWithinGlobalCoordUtil (utility.cpp:170-192; also Session.cpp:186-202, Removerter.cpp:158-177):
 * out = concat_k pose_k * (lidar2base * scan_k), two-step transform with f32 rounding after each step. */
int ltr_merge_scans_global(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, ltr_cloud* out);

/* octreeDownsampling (utility.cpp:204-219): one centroid per occupied voxel, octree depth-first order. */
int ltr_voxel_centroid(ltr_ctx* ctx, ltr_cloud in, float leaf, ltr_cloud* out);
/* Same, applied independently to every keyframe cloud (Session::updateScansScanwise, Session.cpp:374-375). */
int ltr_voxel_centroid_per_keyframe(ltr_ctx* ctx, ltr_scanset in, float leaf, ltr_scanset* out);

/* pcl::VoxelGrid as Session::loadKeyframes applies it to every scan it reads (Session.cpp:284-289), byte-identical to the host restatement
 * voxel_grid_span (lt_mapper_b200/csrc/host/io.cpp): one centroid per occupied voxel in ascending voxel-index order, each summed in the
 * order libstdc++'s std::sort leaves the (index, point) entries.  When the product of the three voxel extents exceeds INT32_MAX the
 * filter takes PCL's overflow exit ("Leaf size is too small for the input dataset") and the scan is returned unchanged; *overflowed
 * (optional) is then 1.  An empty input gives an empty output.  leaf <= 0 or non-finite: LTR_ERR_INVALID. */
int ltr_voxel_grid(ltr_ctx* ctx, ltr_cloud in, float leaf, ltr_cloud* out, int32_t* overflowed);
/* Same, applied to every keyframe of `in` independently (the loadKeyframes loop, Session.cpp:272-303); n_overflowed (optional) receives
 * the number of scans that took the overflow exit. */
int ltr_voxel_grid_per_keyframe(ltr_ctx* ctx, ltr_scanset in, float leaf, ltr_scanset* out, int32_t* n_overflowed);

/* One remove / revert / ND / PD pass == calcDescrepancyAndParseDynamicPointIdxForEachScan{,ForND,ForPD}
 * (Removerter.cpp:542-593, 485-540, 429-482) over the source keyframes [kf_begin, kf_end) of `scans`:
 * scan range image, two-step map transform, map range image + index image, signed diff, threshold,
 * union over keyframes.  The result is the per-map-point dynamic flag array kept on the device
 * (1 = in the reference's dynamic_point_indexes set).  With accumulate != 0 the new flags are OR-ed
 * into the existing ones of the same map (keyframe-sharded multi-GPU: each rank calls with its own
 * keyframe range, then the flag arrays are max-reduced across ranks).
 * n_dynamic (optional) receives the number of flagged points of this context after the pass.
 * The scan-side images of a pass (scan range image, test image, sliding-window maxima) do not depend on the map: the context
 * keeps those of the last two (scan set, poses, keyframe range, image shape) combinations, so a later pass on the same scans at
 * the same resolution does not rebuild them.  They are dropped when the scan set or the poses are freed and by
 * ltr_scan_images_release.  Their two storage blocks are kept for the next sets until ltr_scan_images_release(ctx, 1),
 * ltr_destroy or an allocation that runs out of memory, and never exceed a quarter of the memory the context could still use
 * (environment: LTR_SCAN_IMAGE_CACHE_MB=n caps them at n MiB; 0 builds the images per launch, without keeping them). */
int ltr_remove_pass(ltr_ctx* ctx, ltr_cloud map, ltr_scanset scans, ltr_poses poses, int32_t kf_begin, int32_t kf_end,
                    int32_t mode, float res_alpha, float diff_thres, int32_t accumulate, int64_t* n_dynamic);
/* ltr_remove_pass with the range-adaptive discrepancy threshold the reference leaves commented out in
 * calcDescrepancyAndParseDynamicPointIdx (Removerter.cpp:393-402, line 396 in place of 398): each pixel of each keyframe compares its
 * diff (scan - map for HD / revert / PD, map - scan for ND) with t = fl(adaptive_coeff * s), s the keyframe's scan range at the pixel
 * (10000 without a return), instead of a constant: flagged iff diff < 200 && diff > t.  The winner, the union over keyframes and the
 * kept scan-side images behave as in ltr_remove_pass.  adaptive_coeff must be finite and in (0, 1) (the reference's value is 0.05),
 * else LTR_ERR_INVALID. */
int ltr_remove_pass_adaptive(ltr_ctx* ctx, ltr_cloud map, ltr_scanset scans, ltr_poses poses, int32_t kf_begin, int32_t kf_end,
                             int32_t mode, float res_alpha, float adaptive_coeff, int32_t accumulate, int64_t* n_dynamic);
/* ltr_remove_pass (adaptive_coeff = 0, constant diff_thres) or ltr_remove_pass_adaptive (adaptive_coeff in (0, 1), diff_thres unused) in
 * which keyframe k sees only its ball subset of the map: the points i with d2 < r2, d2 = fl(fl(dx*dx + dy*dy) + dz*dz) in f32 without
 * contraction, dx = fl(x_i - c_k.x), c_k the f32-rounded translation column of poses[k] (not the inverse), r2 = (float)(R*R) in double
 * (takeGlobalMapSubsetWithinBall, Removerter.cpp:415-427, behind kUseSubsetMapCloud / kBallSize, Removerter.h:46-48; FLANN's L2_Simple
 * distance and strict radius test).  A point with a non-finite coordinate is in no ball.  The flags are the OR over k of the
 * single-keyframe pass on the subset, on map indices; the subset keeps map order, so ties between equal ranges in a pixel go to the lowest
 * map index as in ltr_remove_pass.  Modes HD / ND / PD.  ball_radius must be finite and > 0, and adaptive_coeff 0 or in (0, 1), else
 * LTR_ERR_INVALID.  ltr_last_pass_stats counts the pairs outside the balls in [1] (settled without exact arithmetic) and, where a whole
 * 128-point tile is outside a ball, in [6] with the culled pairs; [0] stays K * N. */
int ltr_remove_pass_ball(ltr_ctx* ctx, ltr_cloud map, ltr_scanset scans, ltr_poses poses, int32_t kf_begin, int32_t kf_end,
                         int32_t mode, float res_alpha, float diff_thres, float adaptive_coeff, float ball_radius,
                         int32_t accumulate, int64_t* n_dynamic);
/* Drops the scan-side images ltr_remove_pass keeps; free_storage != 0 also returns their storage to the context's allocator cache. */
int ltr_scan_images_release(ltr_ctx* ctx, int32_t free_storage);
/* Device pointer to the N flag bytes of the last ltr_remove_pass on `map` (for a caller's own all-reduce). */
int ltr_flags_device_ptr(ltr_ctx* ctx, ltr_cloud map, uint8_t** flags, int64_t* n);
int ltr_flags_download(ltr_ctx* ctx, ltr_cloud map, uint8_t* flags, int64_t capacity);
int ltr_flags_upload(ltr_ctx* ctx, ltr_cloud map, const uint8_t* flags, int64_t n);
/* getStaticIdxFromDynamicIdx + parsePointcloudSubsetUsingPtIdx x2 (Removerter.cpp:675-687, 933-946):
 * static = unflagged points, dynamic = flagged points, both in ascending map-index order. */
int ltr_apply_partition(ltr_ctx* ctx, ltr_cloud map, ltr_cloud* out_static, ltr_cloud* out_dynamic);

/* Session::parseScansViaProjection (Session.cpp:348-360) for keyframes [kf_begin, kf_end): project `map`
 * into each keyframe at res_alpha (reference: kReprojectionAlpha = 3.0) and emit, row-major over pixels,
 * the nearest map point of every pixel whose winning index != 0 (utility.cpp:74-89), in that keyframe's
 * LiDAR frame.  out has kf_end - kf_begin keyframes. */
int ltr_parse_projected(ltr_ctx* ctx, ltr_cloud map, ltr_poses poses, int32_t kf_begin, int32_t kf_end, float res_alpha,
                        ltr_scanset* out);

/* Session::extractLowDynPointsViaKnnDiff / extractHighDynPointsViaKnnDiff (Session.cpp:393-427, 487-504) with
 * partition{Low,High}DynamicPointsOfScanByKnn (Session.cpp:537-642): every point of keyframe k (poses index
 * pose_offset + k) is moved to the global frame (as written in the reference: base2lidar first, then the pose),
 * its k nearest SQUARED distances to `target` are averaged ((float)sum_double / float(k)) and compared with thr;
 * |avg| < thr -> coexist else diff; both partitions are moved back with global2local.  Either output may be NULL.
 * With any query point, a target of k or more points with a non-finite coordinate fails with LTR_ERR_UNSUPPORTED. */
int ltr_knn_diff(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, int32_t pose_offset, ltr_cloud target, int32_t k, float thr,
                 ltr_scanset* out_coexist, ltr_scanset* out_diff);
/* Same decision rule for a flat cloud already in the target's frame (no transforms):
 * Session::removeWeakNDMapPointsHavingStrongNDInNear (Session.cpp:452-484). near = |avg| < thr, far = the rest.
 * With any query point, a target of k or more points with a non-finite coordinate fails with LTR_ERR_UNSUPPORTED. */
int ltr_knn_split_cloud(ltr_ctx* ctx, ltr_cloud query, ltr_cloud target, int32_t k, float thr, ltr_cloud* out_near, ltr_cloud* out_far);
/* The same decision rule keyframe by keyframe, the set difference of LT-map change composition (DESIGN.md §5.3): every point of keyframe j
 * of `query` against the points of keyframe j of `target` only (no transforms).  near = |avg| < thr, far = the rest, both in input order
 * within each keyframe; either output may be NULL.  A target keyframe of 0 < n < k points contributes all n (sum still divided by k); an
 * EMPTY target keyframe is not an error here: all its query points are far.  query and target must have the same number of keyframes
 * (LTR_ERR_INVALID), 1 <= k <= 16 (LTR_ERR_UNSUPPORTED), thr finite and > 0 (LTR_ERR_INVALID).  A non-finite coordinate in either input fails
 * with LTR_ERR_UNSUPPORTED before any output exists.  Keyframes go in launches of at most 8192 keyframes and LTR_DELTA_CHUNK_POINTS query +
 * target points (environment; default 2^24, one keyframe at least). */
int ltr_knn_split_per_keyframe(ltr_ctx* ctx, ltr_scanset query, ltr_scanset target, int32_t k, float thr, ltr_scanset* out_near,
                               ltr_scanset* out_far);

/* criteria of ltr_scanside_split */
typedef enum ltr_scanside_criterion {
    LTR_SCANSIDE_MAP = 0,             /* static iff |avg_map| < thr                         (Removerter.cpp:1049-1060) */
    LTR_SCANSIDE_SCAN_MINUS_MAP = 1   /* static iff fabsf(avg_scan - avg_map) < thr, in f32 (Removerter.cpp:1094-1114) */
} ltr_scanside_criterion;

/* Scan-side removal, Removerter::removeDynamicPointsOfScanByKnn (Removerter.cpp:1019-1069, 1071-1123) as
 * scansideRemovalForEachScan (Removerter.cpp:1253-1310) calls it for every keyframe k of `scans` (poses index pose_offset + k):
 * scan_global = local2global(scan_k, pose, lidar2base), the live 3-argument utility.cpp:160-168 (two steps, f32 rounding after
 * each, as ltr_merge_scans_global); every point, in input order, gets
 *   avg_map  = (float)(sum_double of its k smallest SQUARED distances to `map`) / float(k)
 *   avg_scan = the same over scan_global itself (the point is its own first neighbour; duplicates count)
 * with FLANN's L2_Simple distances ((dx*dx + dy*dy) + dz*dz in f32) summed in ascending order; a target of n < k points contributes
 * all n and is still divided by k.  Static and dynamic points keep their input order and are moved back with
 * global2local(..., inv_pose, base2lidar) (utility.cpp:194-202).  Either output may be NULL.
 * 1 <= k <= 16, thr > 0.  An empty map, or a non-finite coordinate in the map or in any scan, fails with LTR_ERR_UNSUPPORTED.
 * Keyframes are processed in launches of at most LTR_SCANSIDE_CHUNK_POINTS points (environment; default 2^24, one keyframe at least). */
int ltr_scanside_split(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, int32_t pose_offset, ltr_cloud map, int32_t criterion,
                       int32_t k, float thr, ltr_scanset* out_static, ltr_scanset* out_dynamic);
/* Counters of the last ltr_scanside_split: [0] points, [1] map searches and [2] own-scan searches that the bounded pass on the finest
 * grid did not settle (they went on to the expanding pass), [3] launches (keyframe chunks). */
int ltr_scanside_stats(ltr_ctx* ctx, int64_t* stats4);

/* ICP refinement of the low-dynamic kNN diff (Session.cpp:393-402, 549-584, switched off in the reference by useICPrefinement):
 * PCL's IterativeClosestPoint control flow with the reference's parameters and arithmetic fixed by this project (DESIGN.md §5.2,
 * lt_mapper_b200/csrc/icp.cu).  ltr_icp_params_default fills the reference's values. */
typedef struct ltr_icp_params {
    double max_correspondence_distance;   /* 150 (setMaxCorrespondenceDistance): pairs with d2 > 150^2 are dropped */
    int32_t max_iterations;               /* 100 (setMaximumIterations), >= 1 */
    double transformation_epsilon;        /* 1e-6 (setTransformationEpsilon): rotation threshold 1 - eps, squared-translation threshold eps */
    double euclidean_fitness_epsilon;     /* 1e-6 (setEuclideanFitnessEpsilon): relative MSE change */
    double mse_threshold_absolute;        /* 1e-12 (DefaultConvergenceCriteria): absolute MSE change */
    int32_t min_correspondences;          /* 3: fewer correspondences stop the loop, not converged */
    float source_leaf;                    /* 0.4 m: octreeDownsampling of each keyframe's global scan (Session.cpp:558-559) */
} ltr_icp_params;
/* exit reasons of ltr_icp_refine (pcl::registration::DefaultConvergenceCriteria::ConvergenceState) */
typedef enum ltr_icp_exit {
    LTR_ICP_ITERATIONS = 1,           /* iterations >= max_iterations */
    LTR_ICP_TRANSFORM = 2,            /* the last increment is below the rotation and translation thresholds */
    LTR_ICP_ABS_MSE = 3,              /* |mse - prev_mse| < mse_threshold_absolute */
    LTR_ICP_REL_MSE = 4,              /* |mse - prev_mse| / prev_mse < euclidean_fitness_epsilon */
    LTR_ICP_NO_CORRESPONDENCES = 5    /* fewer than min_correspondences correspondences (an empty keyframe among them) */
} ltr_icp_exit;
void ltr_icp_params_default(ltr_icp_params* p);
/* Registers every keyframe k of `scans` (poses index pose_offset + k), moved to the global frame as ltr_knn_diff moves it and voxelised
 * per keyframe at source_leaf, to `target_down` (the other session's map at 0.4 m, ltr_voxel_centroid), one CTA per keyframe.  Outputs
 * (host arrays of K entries, each may be NULL): the final float 4x4 (row-major, 16 per keyframe), getFitnessScore() (mean nearest
 * squared distance of the moved source to target_down, DBL_MAX without source points), iterations and the exit reason.  params NULL:
 * the defaults.  An empty target_down or a non-finite coordinate in it or in any moved scan fails with LTR_ERR_UNSUPPORTED.  Keyframes
 * go in launches of at most LTR_ICP_CHUNK_POINTS source points (environment; default 2^24, one keyframe at least). */
int ltr_icp_refine(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, int32_t pose_offset, ltr_cloud target_down, const ltr_icp_params* params,
                   float* T16_out, double* fitness_out, int32_t* iterations_out, int32_t* exit_out);
/* ltr_knn_diff with the refinement applied: the global points of keyframe k with accepted[k] != 0 are moved by T16[16k..16k+16) in f32
 * (((m0 x + m1 y) + m2 z) + m3) before the kNN test against the FULL `target`; both parts go back with global2local, so they hold the
 * registered points.  A keyframe with accepted[k] == 0 gives exactly ltr_knn_diff's bytes.  T16 and accepted are host arrays of K
 * entries (the reference accepts iff fitness < 1.0, Session.cpp:571). */
int ltr_knn_diff_refined(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, int32_t pose_offset, ltr_cloud target, int32_t k, float thr,
                         const float* T16, const uint8_t* accepted, ltr_scanset* out_coexist, ltr_scanset* out_diff);
/* The fine registration of scan-side removal between sessions (removeDynamicPointsOfScanByKnnBtnSession, Removerter.cpp:950-1017, and its
 * isFineRegistration set-up, :1263-1268, 1295-1297, 1325-1331; commented out in the reference): ltr_icp_refine with step 1 replaced by the
 * way ltr_scanside_split moves a scan, local2global(scan_k, pose, lidar2base) (utility.cpp:160-168).  Same arguments, outputs, errors and
 * chunking as ltr_icp_refine; with the identity extrinsic the two return the same bytes. */
int ltr_icp_refine_scanside(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, int32_t pose_offset, ltr_cloud target_down,
                            const ltr_icp_params* params, float* T16_out, double* fitness_out, int32_t* iterations_out, int32_t* exit_out);
/* ltr_scanside_split with the fine registration applied (Removerter.cpp:950-1017 under the accept rule of Session.cpp:571-579): the
 * global points of keyframe k with accepted[k] != 0 are moved by T16[16k..16k+16) in f32 (((m0 x + m1 y) + m2 z) + m3) before the finite
 * check and both searches, so "scan minus map" averages over the registered scan; both parts hold the registered points, moved back with
 * global2local.  A keyframe with accepted[k] == 0 gives exactly ltr_scanside_split's bytes (the commented reference would search with the
 * registered points even then; DESIGN.md §5.4).  T16 and accepted are host arrays of K entries, NULL with K > 0 is LTR_ERR_INVALID; the
 * other errors, the chunking and ltr_scanside_stats are those of ltr_scanside_split. */
int ltr_scanside_split_refined(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, int32_t pose_offset, ltr_cloud map, int32_t criterion,
                               int32_t k, float thr, const float* T16, const uint8_t* accepted, ltr_scanset* out_static,
                               ltr_scanset* out_dynamic);

/* ---- multi-GPU exchange points (NCCL, on the context's stream; libnccl is dlopen'ed at first use) ----------------
 * The path shards by keyframe: every per-keyframe loop of the reference (Removerter.cpp:429-593, Session.cpp:348-427) runs on the
 * rank owning the keyframe.  What crosses ranks: the OR of the per-pass dynamic flags (the reference's set union over scans,
 * Removerter.cpp:588-590), clouds merged over all keyframes in keyframe order (utility.cpp:177-189), and whole maps handed from the
 * ranks of one session to the ranks of the other.  Communicators are small int handles owned by the context. */
int ltr_nccl_unique_id(uint8_t* id128);                       /* ncclGetUniqueId on the calling rank; share the 128 bytes with the others */
int ltr_nccl_init(ltr_ctx* ctx, const uint8_t* id128, int32_t rank, int32_t world, int32_t* comm_out);
int ltr_nccl_split(ltr_ctx* ctx, int32_t comm, int32_t color, int32_t key, int32_t* comm_out);   /* key = parent rank */
int ltr_nccl_info(ltr_ctx* ctx, int32_t comm, int32_t* rank, int32_t* world);
int ltr_nccl_destroy(ltr_ctx* ctx, int32_t comm);
int ltr_nccl_version(int32_t* v);
/* in-place ncclAllReduce(uint8, max) of the dynamic flags of `map` (identical maps on every rank of the communicator) */
int ltr_nccl_allreduce_flags(ltr_ctx* ctx, int32_t comm, ltr_cloud map);
/* out[i] = concatenation over ranks 0..world-1 of each rank's local[i]; one size exchange + ONE grouped send/recv for all clouds */
int ltr_nccl_allgather_clouds(ltr_ctx* ctx, int32_t comm, int32_t count, const ltr_cloud* local, ltr_cloud* out);
/* octreeDownsampling (utility.cpp:204-219) of the rank-ordered concatenation of every rank's `local` cloud (a cloud merged over all
 * keyframes, utility.cpp:177-189), WITHOUT gathering the raw points: all-reduced bounding box, key-prefix ranges of equal population,
 * one exchange of each point to the owner of its range, local voxelisation with the global box, all-gather of the centroid slices.
 * The result (replicated on every rank) is bit-identical to ltr_voxel_centroid of the gathered cloud.  A non-finite coordinate on any
 * rank fails on every rank with LTR_ERR_UNSUPPORTED (as ltr_voxel_centroid), before any rank computes a key. */
int ltr_nccl_voxel_centroid_merged(ltr_ctx* ctx, int32_t comm, ltr_cloud local, float leaf, ltr_cloud* out);
/* n_send clouds go to `peer`, n_recv clouds come from `peer` (the peer calls with the mirrored counts) */
int ltr_nccl_exchange_clouds(ltr_ctx* ctx, int32_t comm, int32_t peer, int32_t n_send, const ltr_cloud* send, int32_t n_recv, ltr_cloud* recv);
int ltr_nccl_allgather_i64(ltr_ctx* ctx, int32_t comm, const int64_t* local, int32_t count, int64_t* out /* world * count */);
int ltr_nccl_max_f64(ltr_ctx* ctx, int32_t comm, double v, double* out);
int ltr_nccl_barrier(ltr_ctx* ctx, int32_t comm);
/* the cudaStream_t every kernel and collective of this context is enqueued on */
void* ltr_stream_handle(ltr_ctx* ctx);

/* ---- introspection for tests / profiling ----------------------------------------------------- */
/* Evaluates the device restatement of cart2sph + pixel index (utility.cpp:38-56, 118-123) for n points. */
int ltr_debug_pixel_index(ltr_ctx* ctx, const float* xyz /* n*3 */, int64_t n, int32_t rows, int32_t cols,
                          int32_t* row, int32_t* col, float* range, float* az, float* el);
/* scan2RangeImg (Removerter.cpp:109-156) of keyframe `kf` exactly as ltr_remove_pass builds it (fast pixel evaluation when the context's
 * fast_path is on): rows*cols floats, 10000.0f = no point.  Lets tests compare the image itself, not only what is derived from it. */
int ltr_debug_scan_rimg(ltr_ctx* ctx, ltr_scanset scans, int32_t kf, float res_alpha, float* rimg /* rows*cols */);
/* The exact k-NN average of ltr_scanside_split's "scan minus map" criterion, (float)(double sum of the k smallest squared distances,
 * ascending) / (float)k, for every point of `query` (taken as global coordinates), in one launch of the same search: self == 0 -> against
 * `target` (avg_map); self != 0 -> keyframe j of `query` against its own points, `target` ignored (avg_scan).  unsettled (may be NULL):
 * the queries the bounded pass on the finest level left over (what ltr_scanside_stats [1] / [2] count).  k outside [1, 16], an empty
 * target, a non-finite coordinate, or more than 8192 keyframes with self set fail with LTR_ERR_UNSUPPORTED. */
int ltr_debug_exact_knn_avg(ltr_ctx* ctx, ltr_scanset query, ltr_cloud target, int32_t self, int32_t k, float* avg /* n */, int64_t* unsettled);
/* The correspondence search of ltr_icp_refine for every point of `query`: d = the smallest f32 L2_Simple squared distance to `target`,
 * idx = the lowest target index at that distance.  Where d is +inf, idx is not specified (ltr_icp_refine drops such pairs).  An empty
 * target or a non-finite coordinate fails with LTR_ERR_UNSUPPORTED. */
int ltr_debug_nearest(ltr_ctx* ctx, ltr_cloud query, ltr_cloud target, float* d /* n */, int32_t* idx /* n */);
/* Fast-path validation: for n map points and one inverse pose, writes per point 8 floats:
 * fast pre-round column, fast pre-round row, fast range, r/rho | reference pre-round column, row, range, fast azimuth [rad];
 * margins4 (optional) = column margin a, column margin b (x r/rho), row margin, relative range margin. */
int ltr_debug_fast_project(ltr_ctx* ctx, const float* xyz /* n*3 */, int64_t n, const double* inv_pose16, float res_alpha,
                           float* out8 /* n*8 */, float* margins4);
/* Exhaustive sweep of the fast path's arctangent polynomials: which = 0 -> every float of [0, 1] through the azimuth polynomial,
 * which = 1 -> every float of [0, 0.5] through the short elevation polynomial; returns max |poly(a) - atan(a)| (atan in double) and
 * the argument where it occurs.  The error budget of the margins (project_fast.cuh) quotes these two numbers. */
int ltr_debug_atan_sweep(ltr_ctx* ctx, int32_t which, double* max_abs_err, float* arg_at_max);
/* margins9 of ltr_debug_margins: column margin a, column margin b (x r/rho), row margin, relative range margin, absolute range margin [m],
 * el_direct flag, the derived (un-inflated) column / row error bounds in pixels at r/rho = 1, and the seam limit [rad]: a fast azimuth
 * with |az| >= it is never certain (half a pixel short of +-pi) */
int ltr_debug_margins(ltr_ctx* ctx, float res_alpha, float* margins9);
/* ltr_nccl_voxel_centroid_merged for `world` simulated ranks in this one context, rank r holding locals[r]: the same rank-local stages,
 * with host reductions for the all-reduces and rank-order concatenations for the point exchange and the final all-gather.  cuts (world - 1
 * entries, may be NULL) receives the first prefix bin of each range after the first, send_counts (world * world, may be NULL) at
 * [r * world + d] the points rank r sends to rank d; both are 0 when every rank is empty.  Errors as ltr_nccl_voxel_centroid_merged. */
int ltr_debug_voxel_distributed(ltr_ctx* ctx, int32_t world, const ltr_cloud* locals /* world */, float leaf, ltr_cloud* out,
                                uint32_t* cuts /* world-1, may be null */, int64_t* send_counts /* world*world, may be null */);
/* resetRimgSize (utility.cpp:222-236) */
void ltr_reset_rimg_size(float vfov, float hfov, float alpha, int32_t* rows, int32_t* cols);
/* Statistics of the last ltr_remove_pass / ltr_parse_projected: [0] (point, keyframe) pairs projected, [1] pairs settled by
 * the fast path alone, [2] pairs that needed exact arithmetic, [3] atomics on the winner image, [4] kernel time of the
 * pass in microseconds (CUDA events), [5] pairs that went through the FULL reference arithmetic, [6] pairs skipped by tile culling
 * (they are included in [1]). */
int ltr_last_pass_stats(ltr_ctx* ctx, double* stats7);
/* Accumulated CUDA-event profile of the dominant kernels since the last reset:
 * [0..3] map-projection kernel of ltr_remove_pass: total microseconds, launches, algorithmic bytes
 *        (sum over launches of keyframes_in_launch * (12 N + N/8), SURVEY.md section 8d), point-projections;
 * [4..7] the same for the projection kernel of ltr_parse_projected (bytes: keyframes * 12 N). */
int ltr_profile_get(ltr_ctx* ctx, double* out8);
int ltr_profile_reset(ltr_ctx* ctx);
/* With LTR_TRACE=1 in the environment every hot entry point is timed on the host between two stream synchronisations;
 * this prints the per-entry-point totals to stderr (and clears them if reset != 0). */
int ltr_trace_dump(ltr_ctx* ctx, int reset);
/* CUDA-event stopwatch on the context's own stream (the stream every kernel of this library is launched on). */
int ltr_timer_start(ltr_ctx* ctx);
int ltr_timer_stop(ltr_ctx* ctx, double* milliseconds);

#ifdef __cplusplus
}
#endif
#endif /* LTR_B200_H_ */
