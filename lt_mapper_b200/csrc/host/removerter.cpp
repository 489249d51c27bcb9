// Host orchestration of the LT-removert / LT-map hot path on top of the device C-ABI (include/ltr_b200.h).
// Statement order follows ltremovert/src/Removerter.cpp and ltremovert/src/Session.cpp (cited per function);
// see removerter.h.  No arithmetic on points happens here.
#include "removerter.h"
#include "io.h"
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <cstdio>
#include <utility>

namespace ltremovert_b200 {

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

#define CK(expr)                                                          \
    do {                                                                  \
        const int rc__ = (expr);                                          \
        if (rc__ != LTR_OK) {                                             \
            if (err.empty()) err = ctx ? ltr_last_error(ctx) : "no context"; \
            return rc__;                                                  \
        }                                                                 \
    } while (0)

struct StageTimer {
    Removerter& R; std::string key; double t0;
    StageTimer(Removerter& r, const char* k) : R(r), key(k) { if (R.ctx) ltr_synchronize(R.ctx); t0 = now_s(); }
    ~StageTimer() { if (R.ctx) ltr_synchronize(R.ctx); R.timing[key] += now_s() - t0; }
};

std::map<std::string, CloudOwner*> Session::cloud_names() {
    return {{"map_global_orig_", &map_global_orig_}, {"map_global_curr_", &map_global_curr_},
            {"map_global_curr_static_", &map_global_curr_static_}, {"map_global_curr_dynamic_", &map_global_curr_dynamic_},
            {"map_global_updated_", &map_global_updated_}, {"map_global_updated_strong_", &map_global_updated_strong_},
            {"map_global_nd_", &map_global_nd_}, {"map_global_nd_strong_", &map_global_nd_strong_}, {"map_global_nd_weak_", &map_global_nd_weak_},
            {"map_global_pd_", &map_global_pd_}, {"map_global_pd_orig_", &map_global_pd_orig_},
            {"map_global_pd_strong_", &map_global_pd_strong_}, {"map_global_pd_weak_", &map_global_pd_weak_}};
}
std::map<std::string, ScanSetOwner*> Session::scanset_names() {
    return {{"keyframe_scans_", &keyframe_scans_}, {"keyframe_scans_static_projected_", &keyframe_scans_static_projected_},
            {"keyframe_scans_dynamic_", &keyframe_scans_dynamic_}, {"scans_knn_coexist_", &scans_knn_coexist_},
            {"scans_knn_diff_", &scans_knn_diff_}, {"keyframe_scans_updated_", &keyframe_scans_updated_},
            {"keyframe_scans_updated_strong_", &keyframe_scans_updated_strong_}, {"keyframe_scans_pd_", &keyframe_scans_pd_},
            {"keyframe_scans_strong_pd_", &keyframe_scans_strong_pd_}, {"keyframe_scans_strong_nd_", &keyframe_scans_strong_nd_},
            {"keyframe_scans_weak_nd_", &keyframe_scans_weak_nd_}, {"scans_static_", &scans_static_}, {"scans_dynamic_", &scans_dynamic_},
            {"composed_pd_", &composed_pd_}, {"composed_nd_", &composed_nd_}, {"keyframe_scans_restored_", &keyframe_scans_restored_}};
}

Removerter::Removerter(const ltrh_params& p) : P(p) {
    central_sess_.sess_type_ = "Central"; central_sess_.id = 0;
    query_sess_.sess_type_ = "Query"; query_sess_.id = 1;
}

int Removerter::fail(int code, const std::string& msg) { err = msg; return code; }

// general 4x4 inverse by cofactors (io.cpp `inverse`, the one implementation in this library); stands in for Eigen's
// kSE3MatExtrinsicLiDARtoPoseBase.inverse() (RosParamServer.cpp:30) and Session.cpp:110
static void invert4x4(const double* m, double* out) {
    Mat4 a;
    std::copy(m, m + 16, a.begin());
    const Mat4 r = inverse(a);
    std::copy(r.begin(), r.end(), out);
}

void invert4x4_public(const double* m, double* out) { invert4x4(m, out); }

int Removerter::init() {
    ltr_config cfg;
    ltr_config_default(&cfg);
    cfg.device = P.device;
    cfg.vfov_deg = P.sequence_vfov;
    cfg.hfov_deg = P.sequence_hfov;
    std::memcpy(cfg.lidar2base, P.ExtrinsicLiDARtoPoseBase, sizeof(cfg.lidar2base));
    bool ident = true;
    for (int i = 0; i < 16; ++i) if (cfg.lidar2base[i] != ((i % 5 == 0) ? 1.0 : 0.0)) ident = false;
    if (ident) std::memcpy(cfg.base2lidar, cfg.lidar2base, sizeof(cfg.base2lidar));
    else invert4x4(cfg.lidar2base, cfg.base2lidar);
    cfg.transform_order = P.transform_order;
    cfg.keyframe_batch = P.keyframe_batch;
    cfg.fast_path = P.fast_path;
    const int rc = ltr_create(&ctx, &cfg);
    ctx_owner_.reset(ctx);
    if (rc != LTR_OK) err = ltr_last_error(nullptr);
    if (const char* e = std::getenv("LTR_DIST_VOXEL_MIN")) dist_voxel_min = std::atoll(e);   // tests force the distributed path on small clouds
    return rc;
}

int Removerter::assign(CloudOwner* dst, ltr_cloud src) {
    ltr_cloud c;
    if (src < 0) { CK(ltr_cloud_alloc(ctx, 0, &c)); }
    else CK(ltr_cloud_copy(ctx, src, &c));
    *dst = CloudOwner(ctx, c);
    return LTR_OK;
}
int Removerter::append(CloudOwner* dst, ltr_cloud src) {
    if (dst->get() < 0) return assign(dst, src);
    if (src < 0) return LTR_OK;
    ltr_cloud c;
    CK(ltr_cloud_concat(ctx, dst->get(), src, &c));
    *dst = CloudOwner(ctx, c);
    return LTR_OK;
}
int Removerter::save(const std::string& name, ltr_cloud c) {
    ltr_cloud copy;
    CK(ltr_cloud_copy(ctx, c, &copy));
    saved[name] = CloudOwner(ctx, copy);
    return LTR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Parallel decomposition (SURVEY.md section 8e).  One process per GPU.
//   * Keyframe sharding: the ranks that own a session hold contiguous keyframe blocks of it (scans + poses) in rank order; every
//     per-keyframe loop of the reference runs on the owner.  Maps are replicated on those ranks; after a pass the per-rank flag
//     arrays are OR-ed (reduce_flags) and every rank applies the same partition / voxelisation, so replicas stay bit-identical.
//     Clouds merged over all keyframes are concatenated in rank == keyframe order (gather_cloud).
//   * Session split (world even, split_sessions): ranks [0, world/2) own the central session, the others the query session.
//     Step 1 of the two sessions (Removerter.cpp:1584 / 1587) and the two halves of Step 2 are independent, so the two groups
//     run them concurrently and the replicated per-pass work (partition, voxelisation) is done once per group, not once per
//     rank.  A map crosses groups exactly where the reference reads the other session's member: rank r hands it to rank
//     r + world/2 (exchange_with_partner), one peer-to-peer transfer per rank pair.
// Transport: the native NCCL entry points of libltr_b200.so (ltr_nccl_*), on the context's stream, no host code in the loop.
// ---------------------------------------------------------------------------------------------------------------
int Removerter::comm_init_nccl(const uint8_t* id128, int rank_, int world_, int split_sessions) {
    if (world_ < 1 || rank_ < 0 || rank_ >= world_) return fail(LTR_ERR_INVALID, "bad rank / world");
    rank = rank_; world = world_;
    split = split_sessions && world >= 2 && world % 2 == 0;
    CK(ltr_nccl_init(ctx, id128, rank, world, &nccl_world));
    if (split) {
        int g;
        CK(ltr_nccl_split(ctx, nccl_world, rank < world / 2 ? 0 : 1, rank, &g));
        nccl_group[0] = nccl_group[1] = g;    // a rank only ever uses the group of the session it owns
        group_world = world / 2;
    } else {
        nccl_group[0] = nccl_group[1] = nccl_world;
        group_world = world;
    }
    return LTR_OK;
}

int Removerter::reduce_flags(ltr_cloud map, const Session& over) {
    if (!sharded()) return LTR_OK;
    return ltr_nccl_allreduce_flags(ctx, nccl_group[over.id], map) == LTR_OK ? LTR_OK : fail(LTR_ERR_CUDA, ltr_last_error(ctx));
}

int Removerter::gather_cloud(const Session& over, CloudOwner* cloud) {
    if (!sharded()) return LTR_OK;
    const ltr_cloud local = cloud->get();
    ltr_cloud g;
    CK(ltr_nccl_allgather_clouds(ctx, nccl_group[over.id], 1, &local, &g));
    *cloud = CloudOwner(ctx, g);
    return LTR_OK;
}

int Removerter::exchange_with_partner(int n_send, const ltr_cloud* send, int n_recv, CloudOwner* recv) {
    if (!split) return fail(LTR_ERR_INVALID, "exchange_with_partner outside session-split mode");
    std::vector<ltr_cloud> got((size_t)n_recv);
    if (ltr_nccl_exchange_clouds(ctx, nccl_world, partner(), n_send, send, n_recv, got.data()) != LTR_OK) return fail(LTR_ERR_CUDA, ltr_last_error(ctx));
    for (int i = 0; i < n_recv; ++i) recv[i] = CloudOwner(ctx, got[i]);
    return LTR_OK;
}

int Removerter::load_session(int sess, const float* xyzi, const int64_t* offsets, const double* poses, const double* inv_poses, int K) {
    ltr_scanset ss;
    CK(ltr_scanset_upload(ctx, xyzi, offsets, K, &ss));
    return load_session_scans(sess, ScanSetOwner(ctx, ss), poses, inv_poses, K);
}

int Removerter::load_session_raw(int sess, const float* xyzi, const int64_t* offsets, const double* poses, const double* inv_poses, int K,
                                 int32_t* n_overflowed) {
    ltr_scanset raw, ss;
    CK(ltr_scanset_upload(ctx, xyzi, offsets, K, &raw));
    ScanSetOwner raw_owner(ctx, raw);
    CK(ltr_voxel_grid_per_keyframe(ctx, raw, P.downsample_voxel_size, &ss, n_overflowed));   // Session.cpp:284-289
    raw_owner.reset();
    return load_session_scans(sess, ScanSetOwner(ctx, ss), poses, inv_poses, K);
}

// the common tail of both loads: the device scan set `ss` and the uploaded poses become the session's keyframes
int Removerter::load_session_scans(int sess, ScanSetOwner ss, const double* poses, const double* inv_poses, int K) {
    Session& S = sess == 0 ? central_sess_ : query_sess_;
    ltr_poses ps;
    CK(ltr_poses_upload(ctx, poses, inv_poses, K, &ps));
    S.keyframe_scans_ = std::move(ss);
    S.keyframe_poses_ = PosesOwner(ctx, ps);
    S.num_keyframes_ = K;
    return LTR_OK;
}

int Removerter::octreeDownsampling(CloudOwner* cloud, float leaf) {
    ltr_cloud v;
    CK(ltr_voxel_centroid(ctx, cloud->get(), leaf, &v));
    *cloud = CloudOwner(ctx, v);
    return LTR_OK;
}

int Removerter::octreeDownsamplingAppended(CloudOwner* cloud, float leaf) {
    int64_t n = 0;
    CK(ltr_cloud_size(ctx, cloud->get(), &n));
    if (!sharded() || n < dist_voxel_min) return octreeDownsampling(cloud, leaf);
    const int g = nccl_group[0];            // the rank's own group (both entries are the same communicator)
    int32_t r = 0, w = 1;
    CK(ltr_nccl_info(ctx, g, &r, &w));
    ltr_cloud part, v;
    CK(ltr_cloud_slice(ctx, cloud->get(), n * r / w, n * (r + 1) / w, &part));
    CloudOwner part_owner(ctx, part);
    CK(ltr_nccl_voxel_centroid_merged(ctx, g, part, leaf, &v));
    part_owner.reset();
    *cloud = CloudOwner(ctx, v);
    return LTR_OK;
}

int Removerter::voxeliseMerged(Session& s, ltr_cloud merged, float leaf, CloudOwner* out) {
    ltr_cloud v;
    CK(sharded() ? ltr_nccl_voxel_centroid_merged(ctx, nccl_group[s.id], merged, leaf, &v) : ltr_voxel_centroid(ctx, merged, leaf, &v));
    *out = CloudOwner(ctx, v);
    return LTR_OK;
}

int Removerter::mergeAndDownsample(Session& s, ltr_scanset scans, float leaf, CloudOwner* out) {
    ltr_cloud m;
    CK(ltr_merge_scans_global(ctx, scans, s.keyframe_poses_.get(), &m));      // this rank's keyframes
    CloudOwner merged(ctx, m);
    return voxeliseMerged(s, m, leaf, out);
}

int Removerter::precleaningKeyframes(float radius) {
    for (Session* s : {&central_sess_, &query_sess_}) {
        if (!owns(*s)) continue;
        ltr_scanset c;
        CK(ltr_preclean(ctx, s->keyframe_scans_.get(), radius, &c));
        s->keyframe_scans_ = ScanSetOwner(ctx, c);
    }
    return LTR_OK;
}

int Removerter::makeGlobalMap(Session& s) {
    // with several ranks the voxelised map comes from the distributed voxeliser (each rank sorts its key range of the ~10^8 raw points);
    // map_global_orig_ keeps its meaning (the merged raw cloud of ALL keyframes) through a gather afterwards, in keyframe == rank order
    ltr_cloud merged;
    CK(ltr_merge_scans_global(ctx, s.keyframe_scans_.get(), s.keyframe_poses_.get(), &merged));   // _sess.mergeScansWithinGlobalCoord() (:218), this rank's keyframes
    CloudOwner orig(ctx, merged), curr;
    CK(voxeliseMerged(s, orig.get(), P.downsample_voxel_size, &curr));                    // :225
    CK(gather_cloud(s, &orig));
    s.map_global_orig_ = std::move(orig);
    s.map_global_curr_ = std::move(curr);
    CK(save("OriginalNoisy" + s.sess_type_ + "MapGlobal", s.map_global_curr_.get()));       // :231
    return LTR_OK;
}
int Removerter::makeGlobalMap() {
    if (owns(central_sess_)) CK(makeGlobalMap(central_sess_));
    if (owns(query_sess_)) CK(makeGlobalMap(query_sess_));
    return LTR_OK;
}

// partitionCurrentMap / ForND / ForPD (:801-828, 771-799, 740-768) and the statements of removeOnce / revertOnce / iremoveOnceForND /
// removeOnceForPD that follow it: the kept side (dynamic for revertOnce, static for the others) replaces its slot, is voxelised and becomes
// the new *map; the other side is appended to its slot and voxelised.  Only the HD passes' appended maps go through the distributed voxeliser.
int Removerter::partitionCurrentMapGeneric(CloudOwner* map, Session& source, ltr_scanset scans, int mode, float res, const char* what,
                                           bool keep_dynamic, CloudOwner* stat, CloudOwner* dyn) {
    int64_t n_map = 0;
    CK(ltr_cloud_size(ctx, map->get(), &n_map));
    // n_dynamic is taken from the partition below (after the cross-rank flag union), so no count is requested here
    if (mapBallRadius_ != 0.0f && mode == LTR_MODE_HD)   // removeOnce / revertOnce on the ball subsets (Removerter.cpp:617-624, commented out)
        CK(ltr_remove_pass_ball(ctx, map->get(), scans, source.keyframe_poses_.get(), 0, source.num_keyframes_, mode, res, 0.1f, adaptiveThresholdCoeff_,
                                mapBallRadius_, 0, nullptr));
    else if (adaptiveThresholdCoeff_ != 0.0f)   // Removerter.cpp:396 in place of :398, for every variant
        CK(ltr_remove_pass_adaptive(ctx, map->get(), scans, source.keyframe_poses_.get(), 0, source.num_keyframes_, mode, res, adaptiveThresholdCoeff_, 0, nullptr));
    else
        CK(ltr_remove_pass(ctx, map->get(), scans, source.keyframe_poses_.get(), 0, source.num_keyframes_, mode, res, 0.1f, 0, nullptr));
    CK(reduce_flags(map->get(), source));
    ltr_cloud st, dy;
    CK(ltr_apply_partition(ctx, map->get(), &st, &dy));
    CloudOwner kept(ctx, st), appended(ctx, dy);
    int64_t n_dyn = 0;
    CK(ltr_cloud_size(ctx, dy, &n_dyn));
    log.push_back(PassLog{what, n_map, n_dyn, -1, -1});

    CloudOwner *kept_slot = stat, *appended_slot = dyn;
    if (keep_dynamic) { std::swap(kept_slot, appended_slot); std::swap(kept, appended); }
    *kept_slot = std::move(kept);
    CK(octreeDownsampling(kept_slot, 0.05f));
    CK(assign(map, kept_slot->get()));
    CK(append(appended_slot, appended.get()));
    appended.reset();
    CK(mode == LTR_MODE_HD ? octreeDownsamplingAppended(appended_slot, 0.05f) : octreeDownsampling(appended_slot, 0.05f));
    CK(ltr_cloud_size(ctx, stat->get(), &log.back().n_static_after));
    CK(ltr_cloud_size(ctx, dyn->get(), &log.back().n_dynamic_after));
    return LTR_OK;
}

// keep static :894-895, voxelise :896, map :899-900, append dynamic :902, voxelise :903
int Removerter::removeOnce(Session& t, Session& s, float res) {
    return partitionCurrentMapGeneric(&t.map_global_curr_, s, s.keyframe_scans_.get(), LTR_MODE_HD, res, "removeOnce", false,
                                      &t.map_global_curr_static_, &t.map_global_curr_dynamic_);
}

// keep dynamic :919-920, voxelise :921, map :924-925, append static :927, voxelise :928
int Removerter::revertOnce(Session& t, Session& s, float res) {
    return partitionCurrentMapGeneric(&t.map_global_curr_, s, s.keyframe_scans_.get(), LTR_MODE_HD, res, "revertOnce", true,
                                      &t.map_global_curr_static_, &t.map_global_curr_dynamic_);
}

// keep strong :843-844, voxelise :845, map :848-849, append weak :851, voxelise :852
int Removerter::iremoveOnceForND(Session& t, Session& s, float res) {
    return partitionCurrentMapGeneric(&t.map_global_nd_, s, s.keyframe_scans_static_projected_.get(), LTR_MODE_ND, res, "iremoveOnceForND", false,
                                      &t.map_global_nd_strong_, &t.map_global_nd_weak_);
}

// keep strong :868-869, voxelise :870, map :873-874, append weak :876, voxelise :878
int Removerter::removeOnceForPD(Session& t, Session& s, float res) {
    return partitionCurrentMapGeneric(&t.map_global_pd_, s, s.keyframe_scans_static_projected_.get(), LTR_MODE_PD, res, "removeOnceForPD", false,
                                      &t.map_global_pd_strong_, &t.map_global_pd_weak_);
}

int Removerter::resetCurrrentMapAsDynamic(Session& s, bool as_dynamic) {
    return assign(&s.map_global_curr_, (as_dynamic ? s.map_global_curr_dynamic_ : s.map_global_curr_static_).get());  // :714-732
}

int Removerter::selfRemovert(Session& s) {
    for (int i = 0; i < P.n_schedule; ++i) {
        if (P.schedule_op[i] == LTRH_OP_REMOVE) {
            CK(removeOnce(s, s, P.schedule_res[i]));
        } else {
            CK(resetCurrrentMapAsDynamic(s, true));
            CK(revertOnce(s, s, P.schedule_res[i]));
            CK(resetCurrrentMapAsDynamic(s, false));
        }
    }
    return LTR_OK;
}

int Removerter::extractHighDynPointsViaKnnDiff(Session& s, ltr_cloud target_map) {
    ltr_scanset di;
    CK(ltr_knn_diff(ctx, s.keyframe_scans_.get(), s.keyframe_poses_.get(), 0, target_map, P.num_nn_points_within, P.dist_nn_points_within, nullptr, &di));
    s.keyframe_scans_dynamic_ = ScanSetOwner(ctx, di);
    return LTR_OK;
}

int Removerter::removeHighDynamicPoints() {
    Session& C = central_sess_;
    Session& Q = query_sess_;
    {
        StageTimer t(*this, "hd_remove");
        if (owns(C)) CK(selfRemovert(C));  // shipped schedule: removeOnce(central, central, 2.5) (:1584)
        if (owns(Q)) CK(selfRemovert(Q));  // shipped schedule: removeOnce(query, query, 2.5)     (:1587)
    }
    if (P.extract_high_dyn_knn) {
        StageTimer t(*this, "hd_knn");
        if (owns(C)) CK(extractHighDynPointsViaKnnDiff(C, C.map_global_curr_static_.get()));  // :1591
        if (owns(Q)) CK(extractHighDynPointsViaKnnDiff(Q, Q.map_global_curr_static_.get()));  // :1592
        CloudOwner c, q;
        if (owns(C)) CK(mergeAndDownsample(C, C.keyframe_scans_dynamic_.get(), 0.05f, &c));  // :1594, :1597
        if (owns(Q)) CK(mergeAndDownsample(Q, Q.keyframe_scans_dynamic_.get(), 0.05f, &q));  // :1595, :1598
        if (owns(C)) { CK(save("central_sess_high_dyn", c.get())); c.reset(); }  // :1600
        if (owns(Q)) { CK(save("query_sess_high_dyn", q.get())); q.reset(); }    // :1601
    }
    if (split) {
        // Step 2 reads the OTHER session's static map (Removerter.cpp:1416, 1418): hand mine to my partner, take theirs
        StageTimer t(*this, "exchange");
        Session& mine = owns(C) ? C : Q;
        Session& other = owns(C) ? Q : C;
        const ltr_cloud send = mine.map_global_curr_static_.get();
        CK(exchange_with_partner(1, &send, 1, &other.map_global_curr_static_));
    }
    return LTR_OK;
}

// Multi-GPU: every rank splits the keyframes of scan_sess it holds (its own block, poses included) and needs no collective: after
// removeHighDynamicPoints every rank holds both sessions' static maps -- replicated over all ranks, or in session-split mode its own
// session's map from Step 1 and the other one from the exchange above.
int Removerter::scansideRemovalForEachScan(Session& map_sess, Session& scan_sess, int criterion, bool isFineRegistration) {
    StageTimer t(*this, "scanside");
    scan_sess.scanside_icp_.clear();
    if (!owns(scan_sess)) return LTR_OK;
    if (map_sess.map_global_curr_static_.get() < 0) return fail(LTR_ERR_INVALID, "scansideRemovalForEachScan: no static map of the " + map_sess.sess_type_ + " session (run Steps 1-2 first)");
    if (scan_sess.keyframe_scans_.get() < 0) return fail(LTR_ERR_INVALID, "scansideRemovalForEachScan: no keyframe scans of the " + scan_sess.sess_type_ + " session");
    ltr_scanset st, dy;
    if (!isFineRegistration) {
        CK(ltr_scanside_split(ctx, scan_sess.keyframe_scans_.get(), scan_sess.keyframe_poses_.get(), 0, map_sess.map_global_curr_static_.get(), criterion,
                              P.num_nn_points_within, P.dist_nn_points_within, &st, &dy));   // :1302-1309
    } else {
        // :1263-1268 / :1325-1331 set up the ICP of Session.cpp:396-402 against the map session's map; :978 keeps the registered scan iff
        // getFitnessScore() < 1.0.  A rejected keyframe is split unregistered (the live rule of Session.cpp:571-579, DESIGN.md §5.4).  The
        // registration reaches scanside_icp_ only with the split that used it: a failed call leaves no stats behind.
        IcpStats reg;
        CK(registerKeyframes(scan_sess, scan_sess.keyframe_scans_.get(), map_sess.map_global_curr_static_.get(), ltr_icp_refine_scanside, &reg));
        CK(ltr_scanside_split_refined(ctx, scan_sess.keyframe_scans_.get(), scan_sess.keyframe_poses_.get(), 0, map_sess.map_global_curr_static_.get(),
                                      criterion, P.num_nn_points_within, P.dist_nn_points_within, reg.T16.data(), reg.accepted.data(), &st, &dy));
        scan_sess.scanside_icp_ = std::move(reg);
    }
    scan_sess.scans_static_ = ScanSetOwner(ctx, st);
    scan_sess.scans_dynamic_ = ScanSetOwner(ctx, dy);
    return LTR_OK;
}

int Removerter::parseScansViaProjection(Session& s, ltr_cloud map, ScanSetOwner* vec_to_store) {
    ltr_scanset out;
    CK(ltr_parse_projected(ctx, map, s.keyframe_poses_.get(), 0, s.num_keyframes_, Session::kReprojectionAlpha, &out));
    *vec_to_store = ScanSetOwner(ctx, out);
    return LTR_OK;
}

int Removerter::parseStaticScansViaProjection() {
    StageTimer t(*this, "parse_static");
    if (owns(central_sess_)) CK(parseScansViaProjection(central_sess_, central_sess_.map_global_curr_.get(), &central_sess_.keyframe_scans_static_projected_));  // Session.cpp:305-308
    if (owns(query_sess_)) CK(parseScansViaProjection(query_sess_, query_sess_.map_global_curr_.get(), &query_sess_.keyframe_scans_static_projected_));
    return LTR_OK;
}

int Removerter::registerKeyframes(Session& s, ltr_scanset scans, ltr_cloud target_map, decltype(&ltr_icp_refine) icp, IcpStats* out) {
    int32_t K = 0;
    int64_t npts = 0;
    CK(ltr_scanset_info(ctx, scans, &K, &npts));
    out->resize((size_t)K);
    ltr_cloud tgt;
    CK(ltr_voxel_centroid(ctx, target_map, 0.4f, &tgt));   // Session.cpp:400
    CloudOwner tgt_owner(ctx, tgt);
    CK(icp(ctx, scans, s.keyframe_poses_.get(), 0, tgt, nullptr, out->T16.data(), out->fitness.data(), out->iterations.data(), out->exit.data()));
    for (int32_t k = 0; k < K; ++k) out->accepted[(size_t)k] = out->fitness[(size_t)k] < 1.0 ? 1 : 0;   // Session.cpp:571
    return LTR_OK;
}

int Removerter::extractLowDynPointsViaKnnDiff(Session& s, ltr_cloud target_map) {
    ltr_scanset co, di;
    s.icp_.clear();
    if (!useICPrefinement_) {
        // Session.cpp:395-402 (0.4 m downsample + ICP target) only feed the refinement, which the reference switches off (Session.cpp:551)
        CK(ltr_knn_diff(ctx, s.keyframe_scans_static_projected_.get(), s.keyframe_poses_.get(), 0, target_map, P.num_nn_points_within, P.dist_nn_points_within, &co, &di));
    } else {
        // Session.cpp:394-402: the ICP target is the other session's map at 0.4 m; partitionLowDynamicPointsOfScanByKnn (:549-584) registers
        // every keyframe to it and keeps the registered scan iff getFitnessScore() < 1.0.  Multi-GPU: this rank's keyframe block against
        // its replica of the target map, no collective.  As in scansideRemovalForEachScan, the stats reach s.icp_ only with the diff.
        IcpStats reg;
        CK(registerKeyframes(s, s.keyframe_scans_static_projected_.get(), target_map, ltr_icp_refine, &reg));
        CK(ltr_knn_diff_refined(ctx, s.keyframe_scans_static_projected_.get(), s.keyframe_poses_.get(), 0, target_map, P.num_nn_points_within,
                                P.dist_nn_points_within, reg.T16.data(), reg.accepted.data(), &co, &di));
        s.icp_ = std::move(reg);
    }
    s.scans_knn_coexist_ = ScanSetOwner(ctx, co);
    s.scans_knn_diff_ = ScanSetOwner(ctx, di);
    return LTR_OK;
}

int Removerter::constructGlobalNDMap(Session& s) {
    CloudOwner m;
    CK(mergeAndDownsample(s, s.scans_knn_diff_.get(), 0.05f, &m));   // Session.cpp:432-434
    s.map_global_nd_ = std::move(m);
    return LTR_OK;
}

int Removerter::constructGlobalPDMap(Session& s) {
    CloudOwner m;
    CK(mergeAndDownsample(s, s.scans_knn_diff_.get(), 0.05f, &m));   // Session.cpp:439-441
    s.map_global_pd_ = std::move(m);
    return assign(&s.map_global_pd_orig_, s.map_global_pd_.get());  // Session.cpp:444
}

int Removerter::removeWeakNDMapPointsHavingStrongNDInNear(Session& s) {
    int64_t n_strong = 0;
    CK(ltr_cloud_size(ctx, s.map_global_nd_strong_.get(), &n_strong));
    if (n_strong == 0) return LTR_OK;  // Session.cpp:454-455
    ltr_cloud near_, far_;
    // hard-coded k = 2, threshold 1.0 (Session.cpp:468-469)
    CK(ltr_knn_split_cloud(ctx, s.map_global_nd_weak_.get(), s.map_global_nd_strong_.get(), 2, 1.0f, &near_, &far_));
    CloudOwner near_owner(ctx, near_), far_owner(ctx, far_);
    CK(append(&s.map_global_nd_strong_, near_));  // Session.cpp:482 (+=)
    near_owner.reset();
    s.map_global_nd_weak_ = std::move(far_owner);  // Session.cpp:483 (=)
    return LTR_OK;
}

int Removerter::filterStrongND(Session& t, Session& s) {
    for (int i = 0; i < 3; ++i) CK(iremoveOnceForND(t, s, 2.5f));  // :1407-1410
    return LTR_OK;
}
int Removerter::filterStrongPD(Session& t, Session& s) {
    for (int i = 0; i < 3; ++i) CK(removeOnceForPD(t, s, 2.5f));   // :1397-1400
    return LTR_OK;
}

// In session-split mode a member lives on the ranks that run the loops producing it:
//   owners of the query keyframes:   filterStrongND (it projects into QUERY keyframes, :1403-1411) -> central map_global_nd_{,strong_,weak_},
//                                    union_map_queryside, pd_map, strong_nd_map, weak_nd_map
//   owners of the central keyframes: filterStrongPD (it projects into CENTRAL keyframes, :1395-1401) -> query map_global_pd_{,strong_,weak_} and the
//                                    central copies (:1434-1436), union_map_centralside, nd_map, strong_pd_map, weak_pd_map
int Removerter::detectLowDynamicPoints() {
    Session& C = central_sess_;
    Session& Q = query_sess_;
    {
        StageTimer t(*this, "ld_knn");
        if (owns(C)) CK(extractLowDynPointsViaKnnDiff(C, Q.map_global_curr_static_.get()));  // :1416
        if (owns(Q)) CK(extractLowDynPointsViaKnnDiff(Q, C.map_global_curr_static_.get()));  // :1418
    }
    {
        StageTimer t(*this, "ld_filter");
        if (owns(C)) CK(constructGlobalNDMap(C));           // :1421
        if (split) {
            // :1427 is independent of :1421-1424, so the query side builds its PD map now and the two maps cross over
            if (owns(Q)) CK(constructGlobalPDMap(Q));
            CloudOwner got;
            // the sender drops its copy: from here on the member lives only where its filter passes run
            if (owns(C)) {
                const ltr_cloud send = C.map_global_nd_.get();
                CK(exchange_with_partner(1, &send, 1, &got));
                C.map_global_nd_.reset();
                Q.map_global_pd_ = std::move(got); CK(assign(&Q.map_global_pd_orig_, Q.map_global_pd_.get()));   // Session.cpp:444
            } else {
                const ltr_cloud send = Q.map_global_pd_.get();
                CK(exchange_with_partner(1, &send, 1, &got));
                Q.map_global_pd_.reset(); Q.map_global_pd_orig_.reset();
                C.map_global_nd_ = std::move(got);
            }
        }
        if (owns(Q)) {
            if (C.map_global_nd_weak_.get() < 0) CK(assign(&C.map_global_nd_weak_, -1));
            CK(filterStrongND(C, Q));                           // :1423
            CK(removeWeakNDMapPointsHavingStrongNDInNear(C));   // :1424
        }
        if (!split) CK(constructGlobalPDMap(Q));                // :1427
        if (owns(C)) {
            if (Q.map_global_pd_weak_.get() < 0) CK(assign(&Q.map_global_pd_weak_, -1));
            CK(filterStrongPD(Q, C));                           // :1429
            // revertStrongPDMapPointsHavingWeakPDInNear: empty TODO in the reference (Session.cpp:447-450)
            CK(assign(&C.map_global_pd_, Q.map_global_pd_.get()));                  // :1434
            CK(assign(&C.map_global_pd_orig_, Q.map_global_pd_orig_.get()));        // :1435
            CK(assign(&C.map_global_pd_strong_, Q.map_global_pd_strong_.get()));    // :1436
        }
    }
    {
        // always-on "save merged maps for visual debug" block (:1442-1480) including its in-place re-downsampling.
        // With several ranks the four merged clouds are voxelised without being gathered (mergeAndDownsample).
        StageTimer t(*this, "ld_merge_viz");
        CloudOwner qco, cco, qdi, cdi;
        if (owns(Q)) CK(mergeAndDownsample(Q, Q.scans_knn_coexist_.get(), 0.05f, &qco));   // :1443-1444
        if (owns(C)) CK(mergeAndDownsample(C, C.scans_knn_coexist_.get(), 0.05f, &cco));   // :1448-1449
        if (owns(Q)) CK(mergeAndDownsample(Q, Q.scans_knn_diff_.get(), 0.05f, &qdi));      // :1453-1454
        if (owns(C)) CK(mergeAndDownsample(C, C.scans_knn_diff_.get(), 0.05f, &cdi));      // :1458-1459
        if (owns(Q)) { CK(save("union_map_queryside", qco.get())); qco.reset(); }     // :1446
        if (owns(C)) { CK(save("union_map_centralside", cco.get())); cco.reset(); }   // :1451
        if (owns(Q)) { CK(save("pd_map", qdi.get())); qdi.reset(); }                  // :1456
        if (owns(C)) { CK(save("nd_map", cdi.get())); cdi.reset(); }                  // :1461
        if (owns(Q)) {   // the ND members live where filterStrongND ran
            int64_t n = 0;
            CK(ltr_cloud_size(ctx, C.map_global_nd_strong_.get(), &n));
            if (n != 0) { CK(octreeDownsampling(&C.map_global_nd_strong_, 0.05f)); CK(save("strong_nd_map", C.map_global_nd_strong_.get())); }   // :1463-1468
            CK(octreeDownsampling(&C.map_global_nd_weak_, 0.05f)); CK(save("weak_nd_map", C.map_global_nd_weak_.get()));                          // :1470-1472
        }
        if (owns(C)) {   // the PD members live where filterStrongPD ran
            CK(octreeDownsampling(&Q.map_global_pd_strong_, 0.05f)); CK(save("strong_pd_map", Q.map_global_pd_strong_.get()));   // :1474-1476
            CK(octreeDownsampling(&Q.map_global_pd_weak_, 0.05f)); CK(save("weak_pd_map", Q.map_global_pd_weak_.get()));         // :1478-1480
        }
    }
    return LTR_OK;
}

int Removerter::updateCurrentMap() {
    Session& C = central_sess_;
    Session& Q = query_sess_;
    CloudOwner uq, uc, upd, strong;
    if (owns(Q)) CK(mergeAndDownsample(Q, Q.scans_knn_coexist_.get(), 0.05f, &uq));  // :1489-1490
    if (split) {
        // Step 3 runs on the owners of the central keyframes; the query side hands over what it holds of the central session
        if (owns(Q)) {
            const ltr_cloud send[3] = {uq.get(), C.map_global_nd_weak_.get(), C.map_global_nd_strong_.get()};
            CK(exchange_with_partner(3, send, 0, nullptr));
            uq.reset();
            return LTR_OK;
        }
        CloudOwner got[3];
        CK(exchange_with_partner(0, nullptr, 3, got));
        uq = std::move(got[0]);
        C.map_global_nd_weak_ = std::move(got[1]);
        C.map_global_nd_strong_ = std::move(got[2]);
    }
    CK(mergeAndDownsample(C, C.scans_knn_coexist_.get(), 0.05f, &uc));  // :1492-1493
    CK(assign(&upd, uq.get()));                       // :1495
    CK(append(&upd, uc.get()));                       // :1496
    CK(append(&upd, C.map_global_nd_weak_.get()));    // :1500
    CK(assign(&strong, upd.get()));                   // :1505
    CK(append(&strong, C.map_global_pd_strong_.get()));  // :1506
    CK(octreeDownsampling(&strong, 0.05f));           // :1507
    CK(append(&upd, C.map_global_pd_orig_.get()));    // :1511
    CK(octreeDownsampling(&upd, 0.05f));              // :1512
    C.map_global_updated_ = std::move(upd); CK(save("updated_map", C.map_global_updated_.get()));                      // :1516-1517
    C.map_global_updated_strong_ = std::move(strong); CK(save("updated_map_strong", C.map_global_updated_strong_.get()));  // :1519-1520
    uq.reset();
    uc.reset();
    return LTR_OK;
}

int Removerter::parseUpdatedStaticScansViaProjection() {
    Session& C = central_sess_;
    if (!owns(C)) return LTR_OK;
    CK(parseScansViaProjection(C, C.map_global_updated_.get(), &C.keyframe_scans_updated_));
    CK(parseScansViaProjection(C, C.map_global_updated_strong_.get(), &C.keyframe_scans_updated_strong_));
    return LTR_OK;
}

int Removerter::parseLDScansViaProjection() {
    Session& C = central_sess_;
    if (!owns(C)) return LTR_OK;
    CK(parseScansViaProjection(C, C.map_global_pd_orig_.get(), &C.keyframe_scans_pd_));
    CK(parseScansViaProjection(C, C.map_global_pd_strong_.get(), &C.keyframe_scans_strong_pd_));
    CK(parseScansViaProjection(C, C.map_global_nd_weak_.get(), &C.keyframe_scans_weak_nd_));
    CK(parseScansViaProjection(C, C.map_global_nd_strong_.get(), &C.keyframe_scans_strong_nd_));
    return LTR_OK;
}

int Removerter::updateScansScanwise() {
    Session& C = central_sess_;
    if (!owns(C)) return LTR_OK;
    ltr_scanset a, b, v;
    CK(ltr_scanset_concat_per_keyframe(ctx, C.keyframe_scans_updated_.get(), C.keyframe_scans_weak_nd_.get(), &a));  // Session.cpp:367-370
    ScanSetOwner a_owner(ctx, a);
    CK(ltr_scanset_concat_per_keyframe(ctx, a, C.keyframe_scans_pd_.get(), &b));                                     // Session.cpp:371
    ScanSetOwner b_owner(ctx, b);
    CK(ltr_voxel_centroid_per_keyframe(ctx, b, 0.05f, &v));                                                          // Session.cpp:374
    a_owner.reset();
    b_owner.reset();
    C.keyframe_scans_updated_ = ScanSetOwner(ctx, v);                                                                // Session.cpp:377
    return LTR_OK;
}

int Removerter::run_step0() {
    StageTimer t(*this, "step0");
    CK(precleaningKeyframes(2.5f));  // run() :1660
    CK(makeGlobalMap());             // run() :1662
    return LTR_OK;
}
int Removerter::run_step12() {
    StageTimer t(*this, "step12");
    CK(removeHighDynamicPoints());        // :1665
    CK(parseStaticScansViaProjection());  // :1666
    CK(detectLowDynamicPoints());         // :1669
    return LTR_OK;
}
int Removerter::run_step3() {
    StageTimer t(*this, "step3");
    CK(updateCurrentMap());                       // :1672
    CK(parseUpdatedStaticScansViaProjection());   // :1673
    CK(parseLDScansViaProjection());              // :1674
    CK(updateScansScanwise());                    // :1675
    return LTR_OK;
}

int Removerter::reset_to_step0() {
    CK(ltr_scan_images_release(ctx, 0));   // their storage stays for the next step's sets
    for (Session* s : {&central_sess_, &query_sess_}) {
        s->icp_.clear();   // Step 2's results
        s->scanside_icp_.clear();
        auto it = saved.find("OriginalNoisy" + s->sess_type_ + "MapGlobal");
        if (!owns(*s)) {   // session-split: everything held of the other session was derived after Step 0
            for (auto& kv : s->cloud_names()) kv.second->reset();
            continue;
        }
        if (it == saved.end()) return fail(LTR_ERR_INVALID, "reset_to_step0: Step 0 has not run");
        for (auto& kv : s->cloud_names()) if (kv.first != "map_global_orig_" && kv.first != "map_global_curr_") kv.second->reset();
        for (auto& kv : s->scanset_names()) if (kv.first != "keyframe_scans_") kv.second->reset();
        CK(assign(&s->map_global_curr_, it->second.get()));
    }
    for (auto it = saved.begin(); it != saved.end();) {
        if (it->first.rfind("OriginalNoisy", 0) == 0) ++it;
        else it = saved.erase(it);
    }
    log.clear();
    timing.clear();
    return LTR_OK;
}

// LT-map cascade (SURVEY.md §8f).  The reference chains sessions through its file protocol: a run's scans_updated/ directory and the
// central pose file are handed to the next run as its central session, where Session::loadKeyframes (Session.cpp:272-303) reads
// each scan back and passes it through pcl::VoxelGrid(downsample_voxel_size).  This does the same in memory and on the device: the
// updated scans (Removerter.cpp:1606-1650, what saveUpdatedScans writes) go through the load-time filter (ltr_voxel_grid_per_keyframe,
// byte-identical to the restatement the file driver used to apply on the host) and become keyframe_scans_ of the central session;
// its poses stay.  Everything derived from the finished pair, and the query session, is released; the caller loads the next query and
// runs Steps 0-3 again.  Ranks that do not own the central session hold none of its scans and only release.
int Removerter::cascade_promote_updated() {
    Session& C = central_sess_;
    if (owns(C) && C.keyframe_scans_updated_.get() < 0) return fail(LTR_ERR_INVALID, "cascade: Step 3 has not run (no keyframe_scans_updated_)");
    ltr_scanset promoted = -1;
    if (owns(C)) CK(ltr_voxel_grid_per_keyframe(ctx, C.keyframe_scans_updated_.get(), P.downsample_voxel_size, &promoted, nullptr));
    ScanSetOwner promoted_owner(ctx, promoted);
    // with delta maps on, this generation's delta (what Step 3 added and removed, in each keyframe's frame) moves out of the session into
    // deltas_ before the release below; ranks without central keyframes hold neither and record an empty pair
    if (deltaMaps_) deltas_.emplace_back(std::move(C.keyframe_scans_pd_), std::move(C.keyframe_scans_strong_nd_));
    for (Session* s : {&central_sess_, &query_sess_}) {
        for (auto& kv : s->cloud_names()) kv.second->reset();
        for (auto& kv : s->scanset_names()) kv.second->reset();
        s->icp_.clear();
        s->scanside_icp_.clear();
    }
    saved.clear();
    query_sess_.keyframe_poses_.reset();
    query_sess_.num_keyframes_ = 0;
    C.keyframe_scans_ = std::move(promoted_owner);
    log.clear();
    timing.clear();
    return LTR_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// LT-map delta maps: change composition and map rollback (DESIGN.md §5.3; the LT-mapper paper's Fig. 10, §IV-C).  Generation g's delta
// is (PD_g, ND_g) = (keyframe_scans_pd_, keyframe_scans_strong_nd_) of the central session after Step 3 of the g-th pair: Step 3 adds
// exactly PD (Session.cpp:362-380) and drops exactly strong ND (Removerter.cpp:1489-1512).  With per-keyframe clouds in each keyframe's
// LiDAR frame, A (-) B = ltr_knn_split_per_keyframe's far part of A against B (num_nn_points_within, dist_nn_points_within),
// V = ltr_voxel_centroid_per_keyframe at 0.05 m, ++ = ltr_scanset_concat_per_keyframe.  Composition over [i, j) starts from
// (PD_i, ND_i) unchanged and folds every further generation g in:
//   ND' = V((ND (-) PD_g) ++ (ND_g (-) PD)),   PD' = V((PD (-) ND_g) ++ (PD_g (-) ND))
// so that removed-then-re-added and added-then-removed points cancel.  Rollback to generation i composes [i, T) over the T recorded
// generations and restores V((L (-) PD) ++ ND) from the live central scans L.  Multi-GPU: each rank works on its own central keyframe
// block; only the restored map's mergeAndDownsample crosses ranks.  Ranks without central keyframes record placeholders and return.
// ---------------------------------------------------------------------------------------------------------------
int Removerter::set_delta_maps(bool on) {
    if (!on) deltas_.clear();
    deltaMaps_ = on;
    return LTR_OK;
}

int Removerter::delta_load(const float* pd_xyzi, const int64_t* pd_off, const float* nd_xyzi, const int64_t* nd_off) {
    if (!deltaMaps_) return fail(LTR_ERR_INVALID, "delta_load: delta maps are off (ltrh_set_delta_maps)");
    std::pair<ScanSetOwner, ScanSetOwner> g;
    if (owns(central_sess_)) {
        if (!pd_off || !nd_off) return fail(LTR_ERR_INVALID, "delta_load: null offsets");
        ltr_scanset pd, nd;
        CK(ltr_scanset_upload(ctx, pd_xyzi, pd_off, central_sess_.num_keyframes_, &pd));
        g.first = ScanSetOwner(ctx, pd);
        CK(ltr_scanset_upload(ctx, nd_xyzi, nd_off, central_sess_.num_keyframes_, &nd));
        g.second = ScanSetOwner(ctx, nd);
    }
    deltas_.push_back(std::move(g));
    return LTR_OK;
}

int Removerter::copy_scanset(ltr_scanset s, ScanSetOwner* out) {
    int32_t K = 0;
    CK(ltr_scanset_info(ctx, s, &K, nullptr));
    const std::vector<int64_t> zero((size_t)K + 1, 0);
    ltr_scanset empty, c;
    CK(ltr_scanset_upload(ctx, nullptr, zero.data(), K, &empty));
    ScanSetOwner empty_owner(ctx, empty);
    CK(ltr_scanset_concat_per_keyframe(ctx, s, empty, &c));
    *out = ScanSetOwner(ctx, c);
    return LTR_OK;
}

int Removerter::set_difference(ltr_scanset a, ltr_scanset b, ScanSetOwner* out) {
    ltr_scanset d;
    CK(ltr_knn_split_per_keyframe(ctx, a, b, P.num_nn_points_within, P.dist_nn_points_within, nullptr, &d));
    *out = ScanSetOwner(ctx, d);
    return LTR_OK;
}

int Removerter::concat_voxelise(ScanSetOwner a, ScanSetOwner b, ScanSetOwner* out) {
    ltr_scanset c, v;
    CK(ltr_scanset_concat_per_keyframe(ctx, a.get(), b.get(), &c));
    a.reset();
    b.reset();
    ScanSetOwner cat(ctx, c);
    CK(ltr_voxel_centroid_per_keyframe(ctx, c, 0.05f, &v));   // Session.cpp:374
    *out = ScanSetOwner(ctx, v);
    return LTR_OK;
}

// (PD, ND) composed over the generations [i, j), i < j; *pd_out and *nd_out are replaced only on success
int Removerter::compose(int i, int j, ScanSetOwner* pd_out, ScanSetOwner* nd_out) {
    ScanSetOwner pd, nd;
    CK(copy_scanset(deltas_[(size_t)i].first.get(), &pd));
    CK(copy_scanset(deltas_[(size_t)i].second.get(), &nd));
    for (int g = i + 1; g < j; ++g) {
        const ltr_scanset pdg = deltas_[(size_t)g].first.get(), ndg = deltas_[(size_t)g].second.get();
        ScanSetOwner a, b, c, d, nd2, pd2;
        CK(set_difference(nd.get(), pdg, &a));
        CK(set_difference(ndg, pd.get(), &b));
        CK(set_difference(pd.get(), ndg, &c));
        CK(set_difference(pdg, nd.get(), &d));
        CK(concat_voxelise(std::move(a), std::move(b), &nd2));
        CK(concat_voxelise(std::move(c), std::move(d), &pd2));
        pd = std::move(pd2);
        nd = std::move(nd2);
    }
    *pd_out = std::move(pd);
    *nd_out = std::move(nd);
    return LTR_OK;
}

int Removerter::compose_changes(int i, int j) {
    if (!deltaMaps_) return fail(LTR_ERR_INVALID, "compose_changes: delta maps are off (ltrh_set_delta_maps)");
    const int T = (int)deltas_.size();
    if (i < 0 || i >= j || j > T) return fail(LTR_ERR_INVALID, "compose_changes: [" + std::to_string(i) + ", " + std::to_string(j) +
                                                               ") is not a non-empty range of the " + std::to_string(T) + " recorded generations");
    Session& C = central_sess_;
    if (!owns(C)) return LTR_OK;
    return compose(i, j, &C.composed_pd_, &C.composed_nd_);
}

int Removerter::rollback(int i) {
    if (!deltaMaps_) return fail(LTR_ERR_INVALID, "rollback: delta maps are off (ltrh_set_delta_maps)");
    const int T = (int)deltas_.size();
    if (i < 0 || i > T) return fail(LTR_ERR_INVALID, "rollback: generation " + std::to_string(i) + " outside [0, " + std::to_string(T) + "]");
    Session& C = central_sess_;
    if (!owns(C)) return LTR_OK;
    if (C.keyframe_scans_.get() < 0) return fail(LTR_ERR_INVALID, "rollback: no central keyframe scans");
    ScanSetOwner restored;
    if (i == T) {
        CK(copy_scanset(C.keyframe_scans_.get(), &restored));
    } else {
        ScanSetOwner pd, nd, kept;
        CK(compose(i, T, &pd, &nd));
        CK(set_difference(C.keyframe_scans_.get(), pd.get(), &kept));
        pd.reset();
        CK(concat_voxelise(std::move(kept), std::move(nd), &restored));
    }
    C.keyframe_scans_restored_ = std::move(restored);
    CloudOwner m;
    CK(mergeAndDownsample(C, C.keyframe_scans_restored_.get(), 0.05f, &m));
    return save("restored_map", m.get());
}

}  // namespace ltremovert_b200

// ---------------------------------------------------------------------------------------------------------------
// flat C view (include/ltr_removert.h)
// ---------------------------------------------------------------------------------------------------------------
using ltremovert_b200::Removerter;
using ltremovert_b200::Session;
using ltremovert_b200::IcpStats;

struct ltrh_removerter { Removerter* R; };
static thread_local std::string g_err;

extern "C" {

void ltrh_params_default(ltrh_params* p) {
    std::memset(p, 0, sizeof(*p));
    p->device = 0;
    p->sequence_vfov = 50.0f;   // RosParamServer.cpp:15
    p->sequence_hfov = 360.0f;  // RosParamServer.cpp:16
    for (int i = 0; i < 16; ++i) p->ExtrinsicLiDARtoPoseBase[i] = (i % 5 == 0) ? 1.0 : 0.0;  // params_ltmapper.yaml:28-31
    p->num_nn_points_within = 2;        // params_ltmapper.yaml:65 (C++ default 3, RosParamServer.cpp:24)
    p->dist_nn_points_within = 0.01f;   // params_ltmapper.yaml:66 (C++ default 0.1, RosParamServer.cpp:25)
    p->downsample_voxel_size = 0.05f;   // RosParamServer.cpp:33
    p->n_schedule = 1;                  // shipped run(): removeOnce(2.5) (Removerter.cpp:1584, 1587)
    p->schedule_op[0] = LTRH_OP_REMOVE;
    p->schedule_res[0] = 2.5f;
    p->extract_high_dyn_knn = 1;
    p->transform_order = 0;
    p->keyframe_batch = 0;
    p->fast_path = 2;
}

int ltrh_create(ltrh_removerter** out, const ltrh_params* p) {
    if (!out || !p) { g_err = "null argument"; return LTR_ERR_INVALID; }
    if (p->n_schedule < 0 || p->n_schedule > LTRH_MAX_SCHEDULE) { g_err = "schedule too long"; return LTR_ERR_INVALID; }
    Removerter* R = new Removerter(*p);
    const int rc = R->init();
    if (rc != LTR_OK) { g_err = R->err; delete R; return rc; }
    *out = new ltrh_removerter{R};
    return LTR_OK;
}
void ltrh_destroy(ltrh_removerter* r) { if (r) { delete r->R; delete r; } }
const char* ltrh_last_error(const ltrh_removerter* r) { return r ? r->R->err.c_str() : g_err.c_str(); }
ltr_ctx* ltrh_context(ltrh_removerter* r) { return r ? r->R->ctx : nullptr; }
int ltrh_comm_init_nccl(ltrh_removerter* r, const uint8_t* id128, int32_t rank, int32_t world, int32_t split_sessions) {
    if (!r || !id128) return LTR_ERR_INVALID;
    r->R->err.clear();
    return r->R->comm_init_nccl(id128, rank, world, split_sessions);
}
// Eigen::Matrix4d::inverse() stand-in (general 4x4 inverse by cofactors) for the inverse keyframe poses of Session.cpp:110
void ltrh_invert_poses(const double* poses16, int32_t K, double* out16) {
    for (int k = 0; k < K; ++k) ltremovert_b200::invert4x4_public(poses16 + 16 * (size_t)k, out16 + 16 * (size_t)k);
}
int ltrh_owns_session(ltrh_removerter* r, int32_t sess) { return r && r->R->owns(sess == 0 ? r->R->central_sess_ : r->R->query_sess_) ? 1 : 0; }

int ltrh_load_session(ltrh_removerter* r, int32_t sess, const float* xyzi, const int64_t* offsets, const double* poses, const double* inv_poses, int32_t K) {
    if (!r || (sess != 0 && sess != 1)) return LTR_ERR_INVALID;
    r->R->err.clear();
    return r->R->load_session(sess, xyzi, offsets, poses, inv_poses, K);
}
int ltrh_load_session_raw(ltrh_removerter* r, int32_t sess, const float* xyzi, const int64_t* offsets, const double* poses, const double* inv_poses, int32_t K) {
    if (!r || (sess != 0 && sess != 1)) return LTR_ERR_INVALID;
    r->R->err.clear();
    return r->R->load_session_raw(sess, xyzi, offsets, poses, inv_poses, K);
}
int ltrh_run_step0(ltrh_removerter* r) { r->R->err.clear(); return r->R->run_step0(); }
int ltrh_run_step12(ltrh_removerter* r) { r->R->err.clear(); return r->R->run_step12(); }
int ltrh_run_step3(ltrh_removerter* r) { r->R->err.clear(); return r->R->run_step3(); }
int ltrh_reset_to_step0(ltrh_removerter* r) { r->R->err.clear(); return r->R->reset_to_step0(); }
int ltrh_cascade_promote_updated(ltrh_removerter* r) { if (!r) return LTR_ERR_INVALID; r->R->err.clear(); return r->R->cascade_promote_updated(); }

int ltrh_set_delta_maps(ltrh_removerter* r, int32_t on) {
    if (!r) return LTR_ERR_INVALID;
    r->R->err.clear();
    return r->R->set_delta_maps(on != 0);
}
int ltrh_delta_load(ltrh_removerter* r, const float* pd_xyzi, const int64_t* pd_off, const float* nd_xyzi, const int64_t* nd_off) {
    if (!r) return LTR_ERR_INVALID;
    r->R->err.clear();
    return r->R->delta_load(pd_xyzi, pd_off, nd_xyzi, nd_off);
}
int32_t ltrh_delta_count(ltrh_removerter* r) { return r ? (int32_t)r->R->deltas_.size() : 0; }
int ltrh_compose_changes(ltrh_removerter* r, int32_t i, int32_t j) {
    if (!r) return LTR_ERR_INVALID;
    r->R->err.clear();
    return r->R->compose_changes(i, j);
}
int ltrh_rollback(ltrh_removerter* r, int32_t i) {
    if (!r) return LTR_ERR_INVALID;
    r->R->err.clear();
    return r->R->rollback(i);
}

int ltrh_scanside_removal(ltrh_removerter* r, int32_t map_sess, int32_t scan_sess, int32_t criterion) {
    if (!r || (map_sess != 0 && map_sess != 1) || (scan_sess != 0 && scan_sess != 1)) return LTR_ERR_INVALID;
    Removerter& R = *r->R;
    R.err.clear();
    return R.scansideRemovalForEachScan(map_sess == 0 ? R.central_sess_ : R.query_sess_, scan_sess == 0 ? R.central_sess_ : R.query_sess_, criterion);
}

int ltrh_scanside_removal_registered(ltrh_removerter* r, int32_t map_sess, int32_t scan_sess, int32_t criterion) {
    if (!r || (map_sess != 0 && map_sess != 1) || (scan_sess != 0 && scan_sess != 1)) return LTR_ERR_INVALID;
    Removerter& R = *r->R;
    R.err.clear();
    return R.scansideRemovalForEachScan(map_sess == 0 ? R.central_sess_ : R.query_sess_, scan_sess == 0 ? R.central_sess_ : R.query_sess_, criterion,
                                        true);
}

int ltrh_set_icp_refinement(ltrh_removerter* r, int32_t on) {
    if (!r) return LTR_ERR_INVALID;
    r->R->useICPrefinement_ = on != 0;
    return LTR_OK;
}

int ltrh_set_adaptive_threshold(ltrh_removerter* r, float c) {
    if (!r || !(c == 0.0f || (c > 0.0f && c < 1.0f))) return LTR_ERR_INVALID;   // NaN fails every comparison
    r->R->adaptiveThresholdCoeff_ = c;
    return LTR_OK;
}

int ltrh_set_map_ball(ltrh_removerter* r, float radius) {
    if (!r || !(radius == 0.0f || (radius > 0.0f && radius <= 3.4028235e38f))) return LTR_ERR_INVALID;   // NaN fails every comparison
    r->R->mapBallRadius_ = radius;
    return LTR_OK;
}

static int copy_icp_stats(const IcpStats& S, int32_t capacity, int32_t* K_out, float* T16, double* fitness, int32_t* iterations,
                          int32_t* exit_reason, uint8_t* accepted) {
    const int32_t K = (int32_t)S.fitness.size();
    *K_out = K;
    if (capacity < K) return LTR_OK;   // a size query
    for (int32_t k = 0; k < K; ++k) {
        if (T16) for (int j = 0; j < 16; ++j) T16[16 * (size_t)k + j] = S.T16[16 * (size_t)k + j];
        if (fitness) fitness[k] = S.fitness[(size_t)k];
        if (iterations) iterations[k] = S.iterations[(size_t)k];
        if (exit_reason) exit_reason[k] = S.exit[(size_t)k];
        if (accepted) accepted[k] = S.accepted[(size_t)k];
    }
    return LTR_OK;
}

int ltrh_icp_stats(ltrh_removerter* r, int32_t sess, int32_t capacity, int32_t* K_out, float* T16, double* fitness, int32_t* iterations,
                   int32_t* exit_reason, uint8_t* accepted) {
    if (!r || (sess != 0 && sess != 1) || !K_out) return LTR_ERR_INVALID;
    const Session& S = sess == 0 ? r->R->central_sess_ : r->R->query_sess_;
    return copy_icp_stats(S.icp_, capacity, K_out, T16, fitness, iterations, exit_reason, accepted);
}

int ltrh_scanside_icp_stats(ltrh_removerter* r, int32_t sess, int32_t capacity, int32_t* K_out, float* T16, double* fitness, int32_t* iterations,
                            int32_t* exit_reason, uint8_t* accepted) {
    if (!r || (sess != 0 && sess != 1) || !K_out) return LTR_ERR_INVALID;
    const Session& S = sess == 0 ? r->R->central_sess_ : r->R->query_sess_;
    return copy_icp_stats(S.scanside_icp_, capacity, K_out, T16, fitness, iterations, exit_reason, accepted);
}

int ltrh_stage(ltrh_removerter* r, const char* name) {
    Removerter& R = *r->R;
    R.err.clear();
    const std::string s(name);
    if (s == "precleaningKeyframes") return R.precleaningKeyframes(2.5f);
    if (s == "makeGlobalMap") return R.makeGlobalMap();
    if (s == "removeHighDynamicPoints") return R.removeHighDynamicPoints();
    if (s == "parseStaticScansViaProjection") return R.parseStaticScansViaProjection();
    if (s == "detectLowDynamicPoints") return R.detectLowDynamicPoints();
    if (s == "updateCurrentMap") return R.updateCurrentMap();
    if (s == "parseUpdatedStaticScansViaProjection") return R.parseUpdatedStaticScansViaProjection();
    if (s == "parseLDScansViaProjection") return R.parseLDScansViaProjection();
    if (s == "updateScansScanwise") return R.updateScansScanwise();
    R.err = "unknown stage " + s;
    return LTR_ERR_INVALID;
}

int ltrh_cloud(ltrh_removerter* r, const char* name, int32_t sess, ltr_cloud* out) {
    Removerter& R = *r->R;
    const std::string n(name);
    if (n.rfind("saved:", 0) == 0) {
        auto it = R.saved.find(n.substr(6));
        if (it == R.saved.end()) { R.err = "no saved cloud " + n; return LTR_ERR_INVALID; }
        *out = it->second.get();
        return LTR_OK;
    }
    Session& S = sess == 0 ? R.central_sess_ : R.query_sess_;
    auto m = S.cloud_names();
    auto it = m.find(n);
    if (it == m.end() || it->second->get() < 0) { R.err = "no cloud " + n; return LTR_ERR_INVALID; }
    *out = it->second->get();
    return LTR_OK;
}
int ltrh_scanset(ltrh_removerter* r, const char* name, int32_t sess, ltr_scanset* out) {
    Removerter& R = *r->R;
    Session& S = sess == 0 ? R.central_sess_ : R.query_sess_;
    auto m = S.scanset_names();
    auto it = m.find(name);
    if (it == m.end() || it->second->get() < 0) { R.err = std::string("no scanset ") + name; return LTR_ERR_INVALID; }
    *out = it->second->get();
    return LTR_OK;
}
double ltrh_timing(ltrh_removerter* r, const char* key) {
    auto it = r->R->timing.find(key);
    return it == r->R->timing.end() ? 0.0 : it->second;
}
int32_t ltrh_log_count(ltrh_removerter* r) { return (int32_t)r->R->log.size(); }
int ltrh_log_get(ltrh_removerter* r, int32_t i, char* what, int32_t cap, int64_t* vals) {
    if (i < 0 || i >= (int32_t)r->R->log.size()) return LTR_ERR_INVALID;
    const auto& l = r->R->log[(size_t)i];
    std::snprintf(what, (size_t)cap, "%s", l.what.c_str());
    vals[0] = l.n_map; vals[1] = l.n_dynamic; vals[2] = l.n_static_after; vals[3] = l.n_dynamic_after;
    return LTR_OK;
}

}  // extern "C"
