/*
 * ltr_removert.h -- host-side orchestrator (libltr_removert.so) that mirrors the reference's
 * ltremovert::Removerter / ltremovert::Session call graph (ltremovert/src/Removerter.cpp:1653-1678,
 * ltremovert/include/removert/Session.h:39-136) on top of the device C-ABI in ltr_b200.h.
 *
 * The C++ classes live in lt_mapper_b200/csrc/host/removerter.{h,cpp}; this header is the flat C view of
 * them used by the Python test/bench harness and by any non-C++ caller.  Sessions are handed over in
 * memory in the form the reference holds them after Session::loadKeyframes (Session.cpp:266-302):
 * per keyframe a cloud of x, y, z, intensity floats plus a pose and its inverse.
 *
 * Multi-GPU: one process per GPU, each owning a contiguous block of keyframes of one or both sessions; maps
 * are replicated on the ranks that own a session.  What crosses ranks (per-pass dynamic-flag union,
 * rank-ordered gather and distributed voxelisation of merged clouds, maps handed between the two session
 * groups) goes through the native NCCL transport of ltr_b200.h (ltr_nccl_*), set up by ltrh_comm_init_nccl.
 */
#ifndef LTR_REMOVERT_H_
#define LTR_REMOVERT_H_

#include "ltr_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ltrh_removerter ltrh_removerter;

#define LTRH_MAX_SCHEDULE 32
enum { LTRH_OP_REMOVE = 0, LTRH_OP_REVERT = 1 };

/* Same keys as the reference's RosParamServer (ltremovert/src/RosParamServer.cpp:4-63). */
typedef struct ltrh_params {
    int32_t device;
    float sequence_vfov, sequence_hfov;          /* removert/sequence_vfov, sequence_hfov */
    double ExtrinsicLiDARtoPoseBase[16];         /* removert/ExtrinsicLiDARtoPoseBase, row-major */
    int32_t num_nn_points_within;                /* kNumKnnPointsToCompare */
    float dist_nn_points_within;                 /* kScanKnnAndMapKnnAvgDiffThreshold (mean SQUARED distance) */
    float downsample_voxel_size;                 /* kDownsampleVoxelSize */
    /* HD-removal schedule: the shipped run() does one removeOnce(2.5) per session (Removerter.cpp:1584,1587);
     * selfRemovert (Removerter.cpp:1378-1393) is {REMOVE r, REVERT 0.95 r, REMOVE r} per resolution r. */
    int32_t n_schedule;
    int32_t schedule_op[LTRH_MAX_SCHEDULE];
    float schedule_res[LTRH_MAX_SCHEDULE];
    int32_t extract_high_dyn_knn;                /* extractHighDynPointsViaKnnDiff in removeHighDynamicPoints (viz output) */
    int32_t transform_order;                     /* see ltr_config */
    int32_t keyframe_batch, fast_path;           /* see ltr_config */
} ltrh_params;

void ltrh_params_default(ltrh_params* p);
int ltrh_create(ltrh_removerter** out, const ltrh_params* p);
void ltrh_destroy(ltrh_removerter* r);
const char* ltrh_last_error(const ltrh_removerter* r);
ltr_ctx* ltrh_context(ltrh_removerter* r);
/* Native multi-GPU transport (ltr_nccl_* of ltr_b200.h; NCCL on the context's stream, no host code in the loop).  id128 = the 128 bytes
 * of ltr_nccl_unique_id() taken on one rank and shared with the others by the launcher.  split_sessions != 0 with an even world:
 * ranks [0, world/2) own the keyframes of the central session, the others those of the query session (each a contiguous block,
 * in rank order); Step 1 of the two sessions and the two halves of Step 2 then run concurrently and a map crosses over exactly
 * where the reference reads the other session's member.  Otherwise every rank owns a block of BOTH sessions.
 * ltrh_load_session on a rank that does not own the session is called with K = 0. */
int ltrh_comm_init_nccl(ltrh_removerter* r, const uint8_t* id128, int32_t rank, int32_t world, int32_t split_sessions);
int ltrh_owns_session(ltrh_removerter* r, int32_t sess);   /* 1 iff this rank holds keyframes of `sess` */

/* Inverse keyframe poses the way the reference obtains them (Session.cpp:110, Eigen::Matrix4d::inverse(): general 4x4 inverse by cofactors).
 * ltrh_load_session takes inverse poses as an INPUT so that every implementation works from identical doubles; callers that do not have the
 * reference's inverses at hand should use this one rather than an LU-based inverse, whose last bits differ. */
void ltrh_invert_poses(const double* poses16, int32_t K, double* out16);

/* sess: 0 = central, 1 = query.  Keyframes are this rank's block (all keyframes when world == 1). */
int ltrh_load_session(ltrh_removerter* r, int32_t sess, const float* xyzi, const int64_t* offsets, const double* poses,
                      const double* inv_poses, int32_t K);
/* The same from the scans as read from disk: Session::loadKeyframes' pcl::VoxelGrid(downsample_voxel_size) (Session.cpp:284-289) runs on
 * the device (ltr_voxel_grid_per_keyframe), then the session is left exactly as ltrh_load_session leaves it with the filtered scans. */
int ltrh_load_session_raw(ltrh_removerter* r, int32_t sess, const float* xyzi, const int64_t* offsets, const double* poses,
                          const double* inv_poses, int32_t K);

/* Removerter::run() split at its step comments (Removerter.cpp:1655-1676) */
int ltrh_run_step0(ltrh_removerter* r);   /* precleaningKeyframes(2.5) + makeGlobalMap            (:1660-1662) */
int ltrh_run_step12(ltrh_removerter* r);  /* removeHighDynamicPoints + parseStaticScansViaProjection + detectLowDynamicPoints (:1665-1669) */
int ltrh_run_step3(ltrh_removerter* r);   /* updateCurrentMap .. updateScansScanwise               (:1672-1675) */
/* Benchmark/test plumbing (not in the reference): restores the state right after Step 0 (map_global_curr_ = the
 * voxelised original map, everything derived freed) so that Step 1+2 can be timed repeatedly; clears log and timings. */
int ltrh_reset_to_step0(ltrh_removerter* r);
/* LT-map cascade (multi-session chaining).  The reference has no call for this: it is done by pointing the next run's
 * central_sess_scan_dir at the previous run's scans_updated/ (written by saveUpdatedScans, Removerter.cpp:1620-1623) with the same
 * central pose file; Session::loadKeyframes (Session.cpp:272-303) then voxel-grids each scan at downsample_voxel_size.  This
 * entry does exactly that in device memory (the scans never leave the GPU) after ltrh_run_step3: central keyframe_scans_ <- VoxelGrid(keyframe_scans_updated_), central poses
 * kept, query session and every derived cloud released, log cleared.  Then ltrh_load_session(r, 1, next query) and run the steps again. */
int ltrh_cascade_promote_updated(ltrh_removerter* r);
/* LT-map delta maps, change composition and map rollback (the LT-mapper paper's Fig. 10, §IV-C; DESIGN.md §5.3).  Off by default.  With
 * on != 0 every later ltrh_cascade_promote_updated records the finished generation's delta (PD_g, ND_g) = (keyframe_scans_pd_,
 * keyframe_scans_strong_nd_) of the central session, per keyframe in that keyframe's LiDAR frame, instead of releasing it.  on == 0 frees
 * the recorded generations (as ltrh_destroy does). */
int ltrh_set_delta_maps(ltrh_removerter* r, int32_t on);
/* Appends one generation from host arrays (what an earlier run wrote to scans_pd/ and scans_nd_strong/): K + 1 offsets each, K = this
 * rank's central keyframes.  Delta maps must be on (LTR_ERR_INVALID otherwise). */
int ltrh_delta_load(ltrh_removerter* r, const float* pd_xyzi, const int64_t* pd_off, const float* nd_xyzi, const int64_t* nd_off);
/* number of recorded generations */
int32_t ltrh_delta_count(ltrh_removerter* r);
/* The changes from generation i to generation j, composed from the deltas [i, j) (0 <= i < j <= count): the central scan sets "composed_pd_"
 * (points added since i) and "composed_nd_" (points removed since i) (ltrh_scanset).  One generation gives its recorded delta unchanged.
 * Delta maps off or a bad range: LTR_ERR_INVALID. */
int ltrh_compose_changes(ltrh_removerter* r, int32_t i, int32_t j);
/* Map rollback: the central scans as of generation i (0 <= i <= count; i == count gives the live scans), restored from the live central
 * keyframe_scans_ and the deltas [i, count) without snapshots: the scan set "keyframe_scans_restored_" and the cloud "saved:restored_map"
 * (merged and voxelised at 0.05 m).  An approximation of the earlier session, as in the paper.  Delta maps off or i outside [0, count]:
 * LTR_ERR_INVALID.  Multi-GPU (this and ltrh_compose_changes): every rank calls; each works on its own central keyframes, the restored
 * map is merged over them, ranks without central keyframes return LTR_OK. */
int ltrh_rollback(ltrh_removerter* r, int32_t i);
/* Removerter::scansideRemovalForEachScan(map_sess, scan_sess) (Removerter.cpp:1253-1310, commented out in the reference; what
 * saveCleanScansPCD asks for): every keyframe of scan_sess held by this rank is split by ltr_scanside_split against map_sess's
 * map_global_curr_static_ with num_nn_points_within / dist_nn_points_within; criterion = ltr_scanside_criterion.  Results: the scan sets
 * "scans_static_" / "scans_dynamic_" of scan_sess (ltrh_scanset).  (C,C) / (Q,Q) clean a session by itself, (C,Q) / (Q,C) give
 * scan-level positive / negative differences.  Valid after ltrh_run_step12 until ltrh_reset_to_step0 or ltrh_cascade_promote_updated
 * (which release the results).  Multi-GPU: each rank splits its own keyframe block; no collective. */
int ltrh_scanside_removal(ltrh_removerter* r, int32_t map_sess, int32_t scan_sess, int32_t criterion);
/* scansideRemovalForEachScan with isFineRegistration (Removerter.cpp:1295-1297; removeDynamicPointsOfScanByKnnBtnSession, :950-1017, both
 * commented out in the reference): every keyframe of scan_sess held by this rank is registered by ltr_icp_refine_scanside (the reference's
 * parameters, ltr_icp_params_default) to ltr_voxel_centroid(map_sess's map_global_curr_static_, 0.4), accepted iff its fitness is below 1.0
 * (:978), and split by ltr_scanside_split_refined against the full static map with num_nn_points_within / dist_nn_points_within.  Results
 * as ltrh_scanside_removal ("scans_static_" / "scans_dynamic_" of scan_sess, the same lifetime), the registration through
 * ltrh_scanside_icp_stats.  Any session pair is accepted; (C,Q) / (Q,C) are the ones the reference registers.  Multi-GPU: each rank
 * registers and splits its own keyframe block against its replica of the map; no collective. */
int ltrh_scanside_removal_registered(ltrh_removerter* r, int32_t map_sess, int32_t scan_sess, int32_t criterion);
/* Session::partitionLowDynamicPointsOfScanByKnn's ICP refinement (Session.cpp:549-584; `useICPrefinement`, false in the reference and by
 * default here).  With on != 0 every later detectLowDynamicPoints (ltrh_run_step12) registers each keyframe to the other session's map at
 * 0.4 m (ltr_icp_refine with the reference's parameters) and runs the kNN diff on the registered scan when its fitness is below 1.0
 * (ltr_knn_diff_refined): scans_knn_coexist_ / scans_knn_diff_ then hold the registered points.  Multi-GPU: each rank refines its own
 * keyframe block against its replica of the target map; no collective. */
int ltrh_set_icp_refinement(ltrh_removerter* r, int32_t on);
/* The range-adaptive discrepancy threshold of calcDescrepancyAndParseDynamicPointIdx (Removerter.cpp:393-402, commented out in the
 * reference): with c in (0, 1) every later remove, revert, ND and PD pass (removeOnce, revertOnce, iremoveOnceForND, removeOnceForPD)
 * runs ltr_remove_pass_adaptive with coefficient c, so that a pixel flags when its diff exceeds fl(c * scan range) instead of 0.1 m; the
 * reference's value is 0.05.  c = 0 (the default) turns it off.  Any other value: LTR_ERR_INVALID.  Multi-GPU: nothing new crosses
 * ranks (the flag union of each pass is unchanged). */
int ltrh_set_adaptive_threshold(ltrh_removerter* r, float c);
/* The reference's ball subset of the map (kUseSubsetMapCloud / kBallSize, Removerter.h:46-48, off there; takeGlobalMapSubsetWithinBall,
 * Removerter.cpp:415-427, called from the HD pass at :617-624): with radius R > 0 every later removeOnce / revertOnce (the selfRemovert
 * schedule of ltrh_run_step12, cascade runs) runs ltr_remove_pass_ball with radius R, so that each keyframe projects only the map points
 * within R of its pose's translation; the adaptive threshold applies when set.  The ND / PD filter passes, the visible-point extraction and
 * Step 3 keep the full map, as the reference does.  The reference's value is 80.  R = 0 (the default) turns it off; any value that is not
 * finite and > 0: LTR_ERR_INVALID.  Multi-GPU: each rank's keyframe block uses its own poses; nothing new crosses ranks. */
int ltrh_set_map_ball(ltrh_removerter* r, float radius);
/* Per-keyframe results of the last refinement of session `sess` on this rank: *K_out keyframes (0 when the last detectLowDynamicPoints ran
 * without refinement, and after ltrh_reset_to_step0 or ltrh_cascade_promote_updated, which release Step 2's results), and, when capacity >= *K_out, the final float 4x4 (16 per keyframe), fitness, iterations, exit reason (ltr_icp_exit)
 * and the accepted flag (fitness < 1.0).  Any array may be NULL. */
int ltrh_icp_stats(ltrh_removerter* r, int32_t sess, int32_t capacity, int32_t* K_out, float* T16, double* fitness, int32_t* iterations,
                   int32_t* exit_reason, uint8_t* accepted);
/* The same for the registration of the last scan-side removal of session `sess`'s scans on this rank (ltrh_scanside_removal_registered):
 * *K_out = 0 when that removal ran without registration (ltrh_scanside_removal), and after ltrh_reset_to_step0 or
 * ltrh_cascade_promote_updated.  Kept apart from ltrh_icp_stats: neither call changes what the other reports. */
int ltrh_scanside_icp_stats(ltrh_removerter* r, int32_t sess, int32_t capacity, int32_t* K_out, float* T16, double* fitness, int32_t* iterations,
                            int32_t* exit_reason, uint8_t* accepted);
/* a single member function of Removerter by name, e.g. "removeHighDynamicPoints" */
int ltrh_stage(ltrh_removerter* r, const char* name);

/* Named device clouds: Session members ("map_global_curr_static_", ...) or what the reference saves as PCD
 * ("saved:pd_map", ...).  Scan sets: per-keyframe members ("keyframe_scans_static_projected_", ...). */
int ltrh_cloud(ltrh_removerter* r, const char* name, int32_t sess, ltr_cloud* out);
int ltrh_scanset(ltrh_removerter* r, const char* name, int32_t sess, ltr_scanset* out);
double ltrh_timing(ltrh_removerter* r, const char* key);  /* seconds spent in a stage (host clock around synchronised calls) */
int32_t ltrh_log_count(ltrh_removerter* r);
/* pass log (the counters the reference prints at Removerter.cpp:811-822, 897, 904): vals = n_map, n_dynamic, n_static_after, n_dynamic_after */
int ltrh_log_get(ltrh_removerter* r, int32_t i, char* what, int32_t cap, int64_t* vals);

/* ---- file-level helpers of the ltremovert node surface (lt_mapper_b200/csrc/host/io.h), used by apps/ltremovert_b200.cpp ---- */
const char* ltrh_io_last_error(void);
/* binary/ascii PCD with float32 x y z [intensity] (pcl::io::loadPCDFile at Session.cpp:275); returns the point count or -1 */
int64_t ltrh_io_read_pcd(const char* path, float* xyzi, int64_t capacity);
/* pcl::io::savePCDFileBinary<PointXYZI>; octree_layout: WIDTH 1 / HEIGHT n as set by octreeDownsampling (utility.cpp:217-218) */
int ltrh_io_write_pcd(const char* path, const float* xyzi, int64_t n, int32_t octree_layout);
/* pose file: one line of 12 or 16 numbers per scan (Session.cpp:102-114); returns the pose count or -1 */
int32_t ltrh_io_read_poses(const char* path, double* poses16, int32_t capacity);
/* Session::parseKeyframes(range, gap) (Session.cpp:138-174, including its skip-two quirk) */
int32_t ltrh_io_parse_keyframes(int32_t num_scans, int32_t start_idx, int32_t end_idx, int32_t gap, int32_t* out, int32_t capacity);
/* Session::parseKeyframesInROI (Session.cpp:230-263, 10 m) */
int32_t ltrh_io_parse_keyframes_in_roi(const double* scan_poses16, int32_t n, const double* roi_poses16, int32_t m, int32_t gap, int32_t* out, int32_t capacity);
/* pcl::VoxelGrid at load (Session.cpp:284-289) incl. the int32 overflow fallback that returns the input unchanged */
int64_t ltrh_io_voxel_grid(const float* xyzi, int64_t n, float leaf, float* out, int64_t capacity, int32_t* overflowed);
/* the same filter over the K scans of a session held back to back (scan k = points [off[k], off[k+1])), scans on different OpenMP
 * threads (Session::loadKeyframes' loop, Session.cpp:272-303).  Returns the total number of output points and fills out_off[K + 1];
 * `out` is written only if capacity (points) suffices. */
int64_t ltrh_io_voxel_grid_scans(const float* xyzi, const int64_t* off, int32_t K, float leaf, float* out, int64_t capacity, int64_t* out_off);
/* one key of a roslaunch-style yaml ("removert/key"): scalar text and/or numeric list */
int ltrh_io_yaml_get(const char* path, const char* key, char* value, int32_t capacity, double* list, int32_t list_capacity, int32_t* list_n);

#ifdef __cplusplus
}
#endif
#endif /* LTR_REMOVERT_H_ */
