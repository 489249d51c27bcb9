// Host-side mirror of ltremovert::Removerter / ltremovert::Session (reference: ltremovert/include/removert/
// Removerter.h:9-204, Session.h:9-136).  Same member and method names, same statement order as
// ltremovert/src/Removerter.cpp / Session.cpp; every cloud is a device handle of the C-ABI in include/ltr_b200.h
// and every loop over keyframes or points is one C-ABI call.  Plain C++17, no CUDA, no ROS/PCL: a ROS build would
// convert pcl::PointCloud<PointXYZI> to/from the float[n][4] arrays at load/save time only.
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>
#include "../../../include/ltr_removert.h"
#include "../handle_owner.h"

namespace ltremovert_b200 {

using ltr::CloudOwner;
using ltr::PosesOwner;
using ltr::ScanSetOwner;

void invert4x4_public(const double* m, double* out);   // general 4x4 inverse by cofactors (removerter.cpp)

struct PassLog { std::string what; int64_t n_map, n_dynamic, n_static_after, n_dynamic_after; };

class Removerter;

// Per-keyframe results of one registration of a session's keyframes on this rank (ltr_icp_refine / ltr_icp_refine_scanside): the final
// float 4x4 (16 per keyframe), fitness, iterations, exit reason and the accept flag (fitness < 1.0)
struct IcpStats {
    std::vector<float> T16;
    std::vector<double> fitness;
    std::vector<int32_t> iterations, exit;
    std::vector<uint8_t> accepted;
    void resize(size_t K) { T16.resize(K * 16); fitness.resize(K); iterations.resize(K); exit.resize(K); accepted.resize(K); }
    void clear() { resize(0); }
};

class Session {
public:
    static constexpr float kReprojectionAlpha = 3.0f;  // Session.h:13
    std::string sess_type_;
    int id = 0;                                        // 0 = central, 1 = query
    int num_keyframes_ = 0;                            // this rank's keyframes
    PosesOwner keyframe_poses_;                        // keyframe_poses_ + keyframe_inverse_poses_ (Session.h:36-37)
    // per-keyframe clouds (Session.h:40-56)
    ScanSetOwner keyframe_scans_, keyframe_scans_static_projected_, keyframe_scans_dynamic_;
    ScanSetOwner scans_knn_coexist_, scans_knn_diff_;
    ScanSetOwner keyframe_scans_updated_, keyframe_scans_updated_strong_, keyframe_scans_pd_, keyframe_scans_strong_pd_, keyframe_scans_strong_nd_,
                 keyframe_scans_weak_nd_;
    // scan-side removal of this session's scans (the commented central_/query_scans_{static,dynamic}_ of Removerter.h)
    ScanSetOwner scans_static_, scans_dynamic_;
    // LT-map change composition (DESIGN.md §5.3) on the central session: the composed delta of ltrh_compose_changes and the scans of
    // ltrh_rollback, per keyframe of this rank
    ScanSetOwner composed_pd_, composed_nd_, keyframe_scans_restored_;
    // ICP refinement of the last extractLowDynPointsViaKnnDiff with useICPrefinement_ on (ltr_icp_refine), per keyframe of this rank
    IcpStats icp_;
    // fine registration of the last scansideRemovalForEachScan of this session's scans with isFineRegistration (ltr_icp_refine_scanside)
    IcpStats scanside_icp_;
    // maps (Session.h:67-87)
    CloudOwner map_global_orig_, map_global_curr_, map_global_curr_static_, map_global_curr_dynamic_;
    CloudOwner map_global_updated_, map_global_updated_strong_;
    CloudOwner map_global_nd_, map_global_nd_strong_, map_global_nd_weak_;
    CloudOwner map_global_pd_, map_global_pd_orig_, map_global_pd_strong_, map_global_pd_weak_;

    std::map<std::string, CloudOwner*> cloud_names();
    std::map<std::string, ScanSetOwner*> scanset_names();
};

class Removerter {
public:
    explicit Removerter(const ltrh_params& p);
    int init();  // creates the device context; returns ltr_status

    // ---- reference call graph (Removerter.cpp) ----
    int precleaningKeyframes(float radius);                                    // :102-106 -> Session.cpp:506-533
    int makeGlobalMap();                                                       // :248-252
    int makeGlobalMap(Session& s);                                             // :213-245
    int removeOnce(Session& target, Session& source, float res);               // :882-905
    int revertOnce(Session& target, Session& source, float res);               // :908-931
    int iremoveOnceForND(Session& target, Session& source, float res);         // :831-854
    int removeOnceForPD(Session& target, Session& source, float res);          // :856-880
    int resetCurrrentMapAsDynamic(Session& s, bool as_dynamic);                // :714-737
    int selfRemovert(Session& s);                                              // :1378-1393 generalised to the configured schedule
    int removeHighDynamicPoints();                                             // :1580-1604
    int parseStaticScansViaProjection();                                       // :1534-1538
    int detectLowDynamicPoints();                                              // :1413-1481
    int filterStrongND(Session& target, Session& source);                      // :1403-1411
    int filterStrongPD(Session& target, Session& source);                      // :1395-1401
    int updateCurrentMap();                                                    // :1483-1524
    int parseUpdatedStaticScansViaProjection();                                // :1551-1561
    int parseLDScansViaProjection();                                           // :1564-1577
    int updateScansScanwise();                                                 // :1540-1548 -> Session.cpp:362-380
    // :1253-1310 (commented out in the reference): scan_sess.scans_{static,dynamic}_ <- removeDynamicPointsOfScanByKnn (:1019-1123) of
    // every keyframe of scan_sess this rank holds, against map_sess.map_global_curr_static_; criterion = ltr_scanside_criterion.
    // isFineRegistration (:1295-1297): each keyframe is first registered to that map at 0.4 m (removeDynamicPointsOfScanByKnnBtnSession,
    // :950-1017) and split registered when its fitness is below 1.0; scan_sess.scanside_icp_ holds the registration.
    int scansideRemovalForEachScan(Session& map_sess, Session& scan_sess, int criterion, bool isFineRegistration = false);
    int run_step0();
    int run_step12();
    int run_step3();
    int reset_to_step0();  // benchmark plumbing, see include/ltr_removert.h
    int cascade_promote_updated();  // LT-map cascade: keyframe_scans_updated_ -> the next run's central keyframe_scans_ (see .cpp)
    // ---- LT-map delta maps (DESIGN.md §5.3; see .cpp) ----
    int set_delta_maps(bool on);
    int delta_load(const float* pd_xyzi, const int64_t* pd_off, const float* nd_xyzi, const int64_t* nd_off);
    int compose_changes(int i, int j);
    int rollback(int i);

    // ---- Session methods (Session.cpp) ----
    int parseScansViaProjection(Session& s, ltr_cloud map, ScanSetOwner* vec_to_store);    // Session.cpp:348-360
    int extractLowDynPointsViaKnnDiff(Session& s, ltr_cloud target_map);                   // Session.cpp:393-427, 549-584
    // every keyframe of `scans` (poses of s) registered by `icp` (ltr_icp_refine or ltr_icp_refine_scanside) to target_map at 0.4 m with
    // the reference's parameters (Session.cpp:396-402); accepted iff fitness < 1.0 (Session.cpp:571)
    int registerKeyframes(Session& s, ltr_scanset scans, ltr_cloud target_map, decltype(&ltr_icp_refine) icp, IcpStats* out);
    int extractHighDynPointsViaKnnDiff(Session& s, ltr_cloud target_map);                  // Session.cpp:487-504
    int constructGlobalNDMap(Session& s);                                                  // Session.cpp:430-435
    int constructGlobalPDMap(Session& s);                                                  // Session.cpp:437-445
    int removeWeakNDMapPointsHavingStrongNDInNear(Session& s);                             // Session.cpp:452-484
    int octreeDownsampling(CloudOwner* cloud, float leaf);                                 // utility.cpp:204-219, in place
    // the same for a freshly appended cloud ("*a += *b", never in octree order): with several ranks every rank contributes its slice of
    // the (replicated) cloud to the distributed voxeliser, so each sorts 1/G of it instead of all of it
    int octreeDownsamplingAppended(CloudOwner* cloud, float leaf);
    // octreeDownsampling of the cloud merged over ALL keyframes of s, given this rank's part `merged` (not consumed): with several
    // ranks the parts are voxelised together without being gathered (ltr_nccl_voxel_centroid_merged)
    int voxeliseMerged(Session& s, ltr_cloud merged, float leaf, CloudOwner* out);
    // mergeScansWithinGlobalCoordUtil (utility.cpp:170-192) followed by octreeDownsampling of the result, the only way the path
    // consumes a merged cloud apart from map_global_orig_
    int mergeAndDownsample(Session& s, ltr_scanset scans, float leaf, CloudOwner* out);

    // ---- plumbing ----
    int load_session(int sess, const float* xyzi, const int64_t* offsets, const double* poses, const double* inv_poses, int K);
    // raw scans as read from disk: Session::loadKeyframes' VoxelGrid(downsample_voxel_size) on the device, then load_session's state;
    // n_overflowed (optional) = scans the filter returned unchanged
    int load_session_raw(int sess, const float* xyzi, const int64_t* offsets, const double* poses, const double* inv_poses, int K,
                         int32_t* n_overflowed = nullptr);
    int assign(CloudOwner* dst, ltr_cloud src);    // "*dst = *src" (deep copy)
    int append(CloudOwner* dst, ltr_cloud src);    // "*dst += *src"
    int save(const std::string& name, ltr_cloud c);  // stands for pcl::io::savePCDFileBinary: keeps a device copy by name
    // ---- multi-GPU (SURVEY.md section 8e; see "Parallel decomposition" in removerter.cpp) ----
    int comm_init_nccl(const uint8_t* id128, int rank, int world, int split_sessions);   // native NCCL transport (ltr_nccl_*)
    bool owns(const Session& s) const { return !split || (rank < world / 2) == (s.id == 0); }
    // the session(s) this rank owns are sharded over more than one rank: flags, merged clouds and appended maps cross ranks
    bool sharded() const { return group_world > 1; }
    int partner() const { return (rank + world / 2) % world; }
    int reduce_flags(ltr_cloud map, const Session& over);               // OR of the dynamic flags over the ranks that own `over`'s keyframes
    int gather_cloud(const Session& over, CloudOwner* cloud);           // *cloud <- rank-ordered concatenation over those ranks
    int exchange_with_partner(int n_send, const ltr_cloud* send, int n_recv, CloudOwner* recv);  // split mode only
    int fail(int code, const std::string& msg);

    // declared first, so that the context is destroyed after every member that owns a handle in it
    std::unique_ptr<ltr_ctx, void (*)(ltr_ctx*)> ctx_owner_{nullptr, ltr_destroy};
    ltr_ctx* ctx = nullptr;   // ctx_owner_.get()
    ltrh_params P;
    bool useICPrefinement_ = false;   // Session.cpp:551 (`bool useICPrefinement { false }`), set by ltrh_set_icp_refinement
    float adaptiveThresholdCoeff_ = 0.0f;   // Removerter.cpp:395-396 (`adaptive_coeff`, commented out); 0: the constant 0.1 (:398), set by ltrh_set_adaptive_threshold
    bool deltaMaps_ = false;   // ltrh_set_delta_maps: cascade_promote_updated records each generation's delta in deltas_
    // per generation (PD_g, ND_g) = (keyframe_scans_pd_, keyframe_scans_strong_nd_) of this rank's central keyframes; empty on ranks
    // without central keyframes, so that every rank counts the same generations
    std::vector<std::pair<ScanSetOwner, ScanSetOwner>> deltas_;
    float mapBallRadius_ = 0.0f;   // Removerter.h:46-48 (`kUseSubsetMapCloud` off, `kBallSize` 80 m); 0: the full map, set by ltrh_set_map_ball
    int rank = 0, world = 1;
    bool split = false;       // session-split: ranks [0, world/2) own the central keyframes, the others the query keyframes
    int nccl_world = -1;      // ltr_nccl communicator handles: everyone, ...
    int nccl_group[2] = {-1, -1};   // ... and the ranks that own session s
    int group_world = 1;      // size of this rank's owner group (1 until comm_init_nccl)
    // appended (replicated) clouds of at least this many points go through the distributed voxeliser, every rank contributing a slice.
    // Off by default: on 4 NVLinked ranks the two size exchanges + the exchange + the gather of a ~10 M point cloud cost more than sorting it on
    // every rank; LTR_DIST_VOXEL_MIN turns it on (the multi-rank tests do).
    int64_t dist_voxel_min = INT64_MAX;
    Session central_sess_, query_sess_;
    std::map<std::string, CloudOwner> saved;
    std::map<std::string, double> timing;
    std::vector<PassLog> log;
    std::string err;

private:
    int load_session_scans(int sess, ScanSetOwner ss, const double* poses, const double* inv_poses, int K);
    int copy_scanset(ltr_scanset s, ScanSetOwner* out);
    int set_difference(ltr_scanset a, ltr_scanset b, ScanSetOwner* out);         // a (-) b: the far part of a against b, per keyframe
    int concat_voxelise(ScanSetOwner a, ScanSetOwner b, ScanSetOwner* out);      // V(a ++ b)
    int compose(int i, int j, ScanSetOwner* pd, ScanSetOwner* nd);
    int partitionCurrentMapGeneric(CloudOwner* map, Session& source, ltr_scanset scans, int mode, float res, const char* what,
                                   bool keep_dynamic, CloudOwner* stat, CloudOwner* dyn);
};

}  // namespace ltremovert_b200
