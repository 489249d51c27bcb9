// ltremovert_b200 -- standalone file-in/file-out driver with the surface of the `removert_removert` ROS node
// (ltremovert/launch/run_ltmapper.launch:6-13, ltremovert/src/removert_main.cpp:3-13): reads the same yaml keys
// (ltremovert/config/params_ltmapper.yaml, namespace "removert"), the same scan directories (binary PCD, fields
// x y z intensity) and pose files (12 numbers per line), runs Removerter::run() (ltremovert/src/Removerter.cpp:1653-1678)
// on the GPU through libltr_removert/libltr_b200, and writes the same output tree (Removerter.cpp:26-50, 231, 1446-1477,
// 1517-1520, 1600-1601, 1607-1650).  No ROS, no PCL; rviz publishing is dropped (side effect only).
//
//   ltremovert_b200 --config params.yaml [--selfremovert] [--pcl110] [--no-split] [--clean-scans[=map|scan-minus-map]]
//                   [--clean-scans-between[=map|scan-minus-map]] [--icp-refinement] [--adaptive-threshold[=c]] [--map-ball[=R]]
//     --selfremovert   run selfRemovert over remove_resolution_list (Removerter.cpp:1378-1393) instead of the shipped
//                      single removeOnce(2.5) (Removerter.cpp:1584, 1587)
//     --pcl110         PCL >= 1.10 transformPointCloud summation order (ltr_config.transform_order = 1)
//     --clean-scans    after Step 3, scansideRemovalForEachScan (C,C) and (Q,Q) (Removerter.cpp:1253-1310, commented out in the reference)
//                      with the "map" criterion (the overload its loop calls, :1306) or "scan-minus-map" (:1071-1123); writes every
//                      keyframe's static / dynamic part to scan_static/<central|query>/ and scan_dynamic/<central|query>/ under the
//                      input scan's name (saveCleanedScans, :1143-1195), and with saveMapPCD the merged, 0.05-voxelised maps of
//                      saveMapPointcloudByMergingCleanedScans (:1197-1251) to map_static/ and map_dynamic/.  Off by default: without it
//                      the output tree is the one the node writes.
//     --clean-scans-between  after Step 3, scansideRemovalForEachScan (C,Q) and (Q,C) with isFineRegistration (Removerter.cpp:1256-1261,
//                      1295-1297; removeDynamicPointsOfScanByKnnBtnSession, :950-1017, commented out in the reference): each keyframe is
//                      registered to the other session's 0.4 m static map and split registered when its fitness is below 1.0, with the
//                      criterion of --clean-scans.  Writes every keyframe's parts under the input scan's name to
//                      scan_static/query_vs_central/ and scan_dynamic/query_vs_central/ (scan-level PD) and scan_static/central_vs_query/
//                      and scan_dynamic/central_vs_query/ (scan-level ND); prints one summary line (keyframes accepted, median
//                      iterations).  Combines with --clean-scans; off by default.
//     --icp-refinement Step 2's kNN diff registers every keyframe to the other session's 0.4 m map first and keeps the registered scan
//                      when its fitness is below 1.0 (partitionLowDynamicPointsOfScanByKnn's `useICPrefinement`, Session.cpp:549-584,
//                      off in the reference); prints one summary line (keyframes accepted, median iterations).  The output tree keeps
//                      its layout; the files derived from Step 2 hold the refined results.
//     --adaptive-threshold  every remove, revert, ND and PD pass flags a pixel when its range diff exceeds fl(c * scan range) instead of
//                      0.1 m (the range-proportional threshold calcDescrepancyAndParseDynamicPointIdx leaves commented out,
//                      Removerter.cpp:393-402); c defaults to the reference's 0.05 and must lie in (0, 1).  Prints one summary line; the
//                      output tree keeps its layout.  There is no yaml key: the reference has none.
//     --compose=<gen_dir>[,<gen_dir>...]  LT-map change composition and map rollback (DESIGN.md §5.3) instead of Steps 0-3: the yaml's central
//                      session (e.g. the last run's scans_updated/ with the central pose file, same keyframe selection and load-time
//                      VoxelGrid) is the live map; the listed output trees of earlier runs, oldest first, give one delta each
//                      (scans_pd/<name>, scans_nd_strong/<name> of every keyframe).  Writes composed/scans_pd/, composed/scans_nd_strong/
//                      (the changes since the first listed run) and composed/scans_restored/ (the central scans as the first listed run
//                      found them) under save_pcd_directory, and with saveMapPCD composed/restored_map.pcd.  The yaml's query session
//                      must still list (its scan directory and pose file are read for the keyframe selection), but none of its scans
//                      is loaded.  The Step 0-3 options (--selfremovert, --clean-scans, --clean-scans-between, --icp-refinement,
//                      --adaptive-threshold, --map-ball) are rejected with it.  Every listed file is checked on every rank before any collective.
//     --map-ball       every removeOnce / revertOnce projects, per keyframe, only the map points within R m of the keyframe's pose (the
//                      reference's kUseSubsetMapCloud / kBallSize, Removerter.h:46-48, off there; takeGlobalMapSubsetWithinBall,
//                      Removerter.cpp:415-427); R defaults to the reference's 80 and must be finite and > 0.  The ND / PD filter passes and
//                      Step 3 keep the full map.  Prints one summary line; the output tree keeps its layout.
//
// Multi-GPU: start one process per GPU with RANK / WORLD_SIZE / LOCAL_RANK in the environment (torchrun, mpirun -x, a shell loop);
// every rank reads the yaml and the pose files, but loads only the scans of ITS keyframe block (even world: ranks < world/2 take the
// central session, the others the query session; --no-split: a block of both).  The NCCL id travels through a file
// ($LTR_NCCL_ID_FILE, default /tmp/ltr_nccl_id_<parent pid>_<MASTER_PORT>).  Maps are written by the first rank of the group that holds
// them, per-keyframe scans by the rank that owns the keyframe; the output tree is the single-process one.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <filesystem>
#include <fstream>
#include <string>
#include <thread>
#include <unistd.h>
#include <vector>
#include "../lt_mapper_b200/csrc/host/io.h"
#include "../lt_mapper_b200/csrc/host/removerter.h"

namespace fs = std::filesystem;
using namespace ltremovert_b200;

static void fsmkdir(const std::string& p) { if (!fs::is_directory(p) || !fs::exists(p)) fs::create_directories(p); }  // Removerter.cpp:6-10

struct LoadedSession {
    SessionFiles files;
    std::vector<std::string> keyframe_names;
    std::vector<float> xyzi;
    std::vector<int64_t> offsets;
    std::vector<double> poses, inv_poses;
};

// the keyframes [k0, k1) of the session's keyframe list (a rank's block; everything in a single-process run), as read from disk:
// Session::loadKeyframes (Session.cpp:266-302) minus its VoxelGrid, which runs on the device (Removerter::load_session_raw)
static bool load_keyframes(LoadedSession& s, size_t k0, size_t k1, std::string* err) {
    s.offsets.assign(1, 0);
    for (size_t kk = k0; kk < k1; ++kk) {
        const int idx = s.files.keyframe_idx[kk];
        HostCloud pts;
        if (!read_pcd(s.files.scan_paths[(size_t)idx], &pts, err)) return false;
        const float* f = reinterpret_cast<const float*>(pts.data());
        s.xyzi.insert(s.xyzi.end(), f, f + 4 * pts.size());
        s.offsets.push_back(s.offsets.back() + (int64_t)pts.size());
        s.keyframe_names.push_back(s.files.scan_names[(size_t)idx]);
        const Mat4& P = s.files.scan_poses[(size_t)idx];
        const Mat4& IP = s.files.scan_inverse_poses[(size_t)idx];
        s.poses.insert(s.poses.end(), P.begin(), P.end());
        s.inv_poses.insert(s.inv_poses.end(), IP.begin(), IP.end());
    }
    return true;
}

static bool save_cloud(Removerter& R, const CloudOwner& h, const std::string& path, bool octree_layout) {
    int64_t n = 0;
    if (ltr_cloud_size(R.ctx, h.get(), &n) != LTR_OK) return false;
    std::vector<float> buf((size_t)n * 4 + 4);
    if (ltr_cloud_download(R.ctx, h.get(), buf.data(), n, &n) != LTR_OK) return false;
    HostCloud c((size_t)n);
    if (n) std::memcpy(c.data(), buf.data(), (size_t)n * 16);
    std::string err;
    if (!write_pcd_binary(path, c, octree_layout, &err)) { std::fprintf(stderr, "%s\n", err.c_str()); return false; }
    return true;
}

static bool save_scans(Removerter& R, const ScanSetOwner& s, const std::vector<std::string>& names, const std::string& dir, bool octree_layout) {  // saveScans (:1632-1650)
    int32_t K = 0; int64_t total = 0;
    if (s.get() < 0 || ltr_scanset_info(R.ctx, s.get(), &K, &total) != LTR_OK) return false;
    std::vector<float> buf((size_t)total * 4 + 4);
    std::vector<int64_t> off((size_t)K + 1);
    if (ltr_scanset_download(R.ctx, s.get(), buf.data(), total, off.data()) != LTR_OK) return false;
    for (int k = 0; k < K; ++k) {
        HostCloud c((size_t)(off[k + 1] - off[k]));
        if (!c.empty()) std::memcpy(c.data(), buf.data() + 4 * off[k], c.size() * 16);
        std::string err;
        if (!write_pcd_binary(dir + "/" + names[(size_t)k], c, octree_layout, &err)) { std::fprintf(stderr, "%s\n", err.c_str()); return false; }
    }
    return true;
}

static int env_int(const char* name, int dflt) { const char* v = std::getenv(name); return v && *v ? std::atoi(v) : dflt; }

// the 128 bytes of ncclGetUniqueId from rank 0 to everybody else, through a file that appears atomically (write + rename)
static bool share_nccl_id(int rank, unsigned char id[128]) {
    const char* e = std::getenv("LTR_NCCL_ID_FILE");
    const char* port = std::getenv("MASTER_PORT");
    const std::string path = e && *e ? e : "/tmp/ltr_nccl_id_" + std::to_string((long)getppid()) + "_" + (port ? port : "0");
    if (rank == 0) {
        if (ltr_nccl_unique_id(id) != LTR_OK) return false;
        { std::ofstream f(path + ".tmp", std::ios::binary); f.write((const char*)id, 128); if (!f) return false; }
        return std::rename((path + ".tmp").c_str(), path.c_str()) == 0;
    }
    for (int tries = 0; tries < 600; ++tries) {   // up to 60 s
        std::ifstream f(path, std::ios::binary);
        if (f && f.read((char*)id, 128) && f.gcount() == 128) return true;
        std::this_thread::sleep_for(std::chrono::milliseconds(100));
    }
    return false;
}

int main(int argc, char** argv) {
    std::string cfg_path;
    bool selfremovert = false, pcl110 = false, no_split = false;
    int clean_scans = -1;   // -1 off, else ltr_scanside_criterion
    int clean_between = -1;   // the same for the registered (C,Q) / (Q,C) removal
    bool icp_refinement = false;
    float adaptive_c = 0.0f;   // 0: the constant threshold
    float ball_r = 0.0f;       // 0: the full map
    const char* usage = "usage: %s --config params.yaml [--selfremovert] [--pcl110] [--no-split] [--clean-scans[=map|scan-minus-map]]"
                        " [--clean-scans-between[=map|scan-minus-map]] [--icp-refinement]"
                        " [--adaptive-threshold[=c], 0 < c < 1] [--map-ball[=R], R > 0] [--compose=<gen_dir>[,<gen_dir>...]]\n";
    std::vector<std::string> compose_dirs;   // --compose: output trees of earlier runs, oldest first
    for (int i = 1; i < argc; ++i) {
        if (!std::strcmp(argv[i], "--config") && i + 1 < argc) cfg_path = argv[++i];
        else if (!std::strcmp(argv[i], "--selfremovert")) selfremovert = true;
        else if (!std::strcmp(argv[i], "--pcl110")) pcl110 = true;
        else if (!std::strcmp(argv[i], "--no-split")) no_split = true;
        else if (!std::strcmp(argv[i], "--clean-scans") || !std::strcmp(argv[i], "--clean-scans=map")) clean_scans = LTR_SCANSIDE_MAP;
        else if (!std::strcmp(argv[i], "--clean-scans=scan-minus-map")) clean_scans = LTR_SCANSIDE_SCAN_MINUS_MAP;
        else if (!std::strcmp(argv[i], "--clean-scans-between") || !std::strcmp(argv[i], "--clean-scans-between=map")) clean_between = LTR_SCANSIDE_MAP;
        else if (!std::strcmp(argv[i], "--clean-scans-between=scan-minus-map")) clean_between = LTR_SCANSIDE_SCAN_MINUS_MAP;
        else if (!std::strcmp(argv[i], "--icp-refinement")) icp_refinement = true;
        else if (!std::strcmp(argv[i], "--adaptive-threshold")) adaptive_c = 0.05f;
        else if (!std::strcmp(argv[i], "--map-ball")) ball_r = 80.0f;
        else if (!std::strncmp(argv[i], "--map-ball=", 11)) {
            char* end = nullptr;
            ball_r = std::strtof(argv[i] + 11, &end);
            if (end == argv[i] + 11 || *end || !(ball_r > 0.0f && ball_r <= 3.4028235e38f)) { std::fprintf(stderr, usage, argv[0]); return 2; }
        }
        else if (!std::strncmp(argv[i], "--compose=", 10)) {
            std::string list = argv[i] + 10;
            for (size_t a = 0; a <= list.size();) {
                const size_t b = std::min(list.find(',', a), list.size());
                if (b == a) { std::fprintf(stderr, usage, argv[0]); return 2; }
                std::string d = list.substr(a, b - a);
                if (d.back() != '/') d += "/";
                compose_dirs.push_back(d);
                a = b + 1;
            }
        }
        else if (!std::strncmp(argv[i], "--adaptive-threshold=", 21)) {
            char* end = nullptr;
            adaptive_c = std::strtof(argv[i] + 21, &end);
            if (end == argv[i] + 21 || *end || !(adaptive_c > 0.0f && adaptive_c < 1.0f)) { std::fprintf(stderr, usage, argv[0]); return 2; }
        }
        else { std::fprintf(stderr, usage, argv[0]); return 2; }
    }
    if (cfg_path.empty()) { std::fprintf(stderr, usage, argv[0]); return 2; }
    if (!compose_dirs.empty() && (selfremovert || clean_scans >= 0 || clean_between >= 0 || icp_refinement || adaptive_c != 0.0f || ball_r != 0.0f)) {
        std::fprintf(stderr, "--compose runs no Step 0-3: --selfremovert, --clean-scans, --clean-scans-between, --icp-refinement, "
                             "--adaptive-threshold and --map-ball cannot be combined with it\n");
        return 2;
    }
    const int rank = env_int("RANK", 0), world = std::max(1, env_int("WORLD_SIZE", 1));
    const bool split = world >= 2 && world % 2 == 0 && !no_split;
    YamlParams y;
    std::string err;
    if (!y.load(cfg_path, &err)) { std::fprintf(stderr, "%s\n", err.c_str()); return 1; }

    // RosParamServer.cpp:4-63 (same keys, same C++ defaults)
    ltrh_params P;
    ltrh_params_default(&P);
    P.device = env_int("LOCAL_RANK", 0);
    P.sequence_vfov = (float)y.num("removert/sequence_vfov", 50.0);
    P.sequence_hfov = (float)y.num("removert/sequence_hfov", 360.0);
    P.num_nn_points_within = (int)y.num("removert/num_nn_points_within", 3);
    P.dist_nn_points_within = (float)y.num("removert/dist_nn_points_within", 0.1);
    P.downsample_voxel_size = (float)y.num("removert/downsample_voxel_size", 0.05);
    const std::vector<double> ext = y.list("removert/ExtrinsicLiDARtoPoseBase");
    if (ext.size() == 16) for (int i = 0; i < 16; ++i) P.ExtrinsicLiDARtoPoseBase[i] = ext[(size_t)i];
    P.transform_order = pcl110 ? 1 : 0;
    const std::vector<double> remove_res = y.list("removert/remove_resolution_list");
    if (selfremovert) {
        P.n_schedule = 0;
        for (double r : remove_res) {   // selfRemovert (Removerter.cpp:1380-1389)
            if (P.n_schedule + 3 > LTRH_MAX_SCHEDULE) break;
            P.schedule_op[P.n_schedule] = LTRH_OP_REMOVE; P.schedule_res[P.n_schedule++] = (float)r;
            P.schedule_op[P.n_schedule] = LTRH_OP_REVERT; P.schedule_res[P.n_schedule++] = (float)(0.95 * (float)r);
            P.schedule_op[P.n_schedule] = LTRH_OP_REMOVE; P.schedule_res[P.n_schedule++] = (float)r;
        }
    }
    std::string save_dir = y.str("removert/save_pcd_directory", "/");
    if (save_dir.empty() || save_dir.back() != '/') save_dir += "/";      // Removerter.cpp:26-27
    const bool save_map_pcd = y.boolean("removert/saveMapPCD", false);
    const int start_idx = (int)y.num("removert/start_idx", 1), end_idx = (int)y.num("removert/end_idx", 100);
    const int keyframe_gap = (int)y.num("removert/keyframe_gap", 10);

    // output tree (Removerter.cpp:28-50)
    const bool compose = !compose_dirs.empty();
    fsmkdir(save_dir);
    const std::string d_updated = save_dir + "scans_updated", d_updated_strong = save_dir + "scans_updated_strong", d_pd = save_dir + "scans_pd",
                      d_pd_strong = save_dir + "scans_pd_strong", d_nd_strong = save_dir + "scans_nd_strong";
    if (!compose)
        for (const std::string& d : {d_updated, d_updated_strong, d_pd, d_pd_strong, d_nd_strong, save_dir + "map_static", save_dir + "map_dynamic"}) fsmkdir(d);

    // Step 0 host side: loadSessionInfo, parseKeyframes, loadKeyframes (run() :1656-1659)
    LoadedSession C, Q;
    if (!list_session(y.str("removert/central_sess_scan_dir", ""), y.str("removert/central_sess_pose_path", ""), &C.files, &err) ||
        !list_session(y.str("removert/query_sess_scan_dir", ""), y.str("removert/query_sess_pose_path", ""), &Q.files, &err)) {
        std::fprintf(stderr, "%s\n", err.c_str());
        return 1;
    }
    if (rank == 0) std::printf(" Total : %zu / %zu scans in the directories.\n", C.files.scan_paths.size(), Q.files.scan_paths.size());
    C.files.keyframe_idx = parse_keyframes((int)C.files.scan_paths.size(), start_idx, end_idx, keyframe_gap);            // Removerter.cpp:92
    std::vector<Mat4> roi;
    for (int i : C.files.keyframe_idx) roi.push_back(C.files.scan_poses[(size_t)i]);
    Q.files.keyframe_idx = parse_keyframes_in_roi(Q.files.scan_poses, roi, keyframe_gap);                               // Removerter.cpp:93
    if (rank == 0)
        std::printf(" Total %zu central keyframes from the index range [%d, %d], %zu query keyframes in the map's ROI\n",
                    C.files.keyframe_idx.size(), start_idx, end_idx, Q.files.keyframe_idx.size());
    // this rank's contiguous keyframe block of each session (keyframe order == rank order); everything when world == 1
    auto block = [&](size_t K, bool owns, size_t* k0, size_t* k1) {
        const int g = split ? world / 2 : world, r = split ? rank % (world / 2) : rank;
        *k0 = owns ? K * (size_t)r / (size_t)g : 0;
        *k1 = owns ? K * (size_t)(r + 1) / (size_t)g : 0;
    };
    const bool owns_c = !split || rank < world / 2, owns_q = !split || rank >= world / 2;
    size_t c0, c1, q0, q1;
    block(C.files.keyframe_idx.size(), owns_c, &c0, &c1);
    block(Q.files.keyframe_idx.size(), owns_q && !compose, &q0, &q1);   // composition needs no query session
    if (!load_keyframes(C, c0, c1, &err) || !load_keyframes(Q, q0, q1, &err)) { std::fprintf(stderr, "%s\n", err.c_str()); return 1; }
    // --compose: one generation per listed tree, what its Step 3 added (scans_pd/) and removed (scans_nd_strong/) in each of this rank's
    // keyframes; read before any collective, so that a missing file stops every rank (agreed below) instead of leaving the others waiting
    std::vector<std::vector<float>> delta_pts;
    std::vector<std::vector<int64_t>> delta_off;
    std::string delta_bad;
    for (const std::string& g : compose_dirs) {
        for (const char* sub : {"scans_pd/", "scans_nd_strong/"}) {
            delta_pts.emplace_back();
            delta_off.emplace_back(1, 0);
            for (const std::string& name : C.keyframe_names) {
                const std::string path = g + sub + name;
                HostCloud pts;
                if (delta_bad.empty() && (!fs::exists(path) || !read_pcd(path, &pts, &err))) delta_bad = path;
                if (!delta_bad.empty()) break;
                const float* f = reinterpret_cast<const float*>(pts.data());
                delta_pts.back().insert(delta_pts.back().end(), f, f + 4 * pts.size());
                delta_off.back().push_back(delta_off.back().back() + (int64_t)pts.size());
            }
        }
    }
    if (!delta_bad.empty()) std::fprintf(stderr, "[rank %d] cannot read delta scan %s\n", rank, delta_bad.c_str());
    if (!delta_bad.empty() && world == 1) return 1;

    Removerter R(P);
    if (R.init() != LTR_OK) { std::fprintf(stderr, "GPU context: %s\n", R.err.c_str()); return 1; }
    auto ck = [&](int rc, const char* what) { if (rc != LTR_OK) { std::fprintf(stderr, "[rank %d] %s failed (%d): %s\n", rank, what, rc, R.err.c_str()); std::exit(1); } };
    if (world > 1) {
        unsigned char id[128];
        if (!share_nccl_id(rank, id)) { std::fprintf(stderr, "[rank %d] could not exchange the NCCL id\n", rank); return 1; }
        ck(R.comm_init_nccl(id, rank, world, split ? 1 : 0), "NCCL init");
    }
    // upload the raw scans; loadKeyframes' VoxelGrid(downsample_voxel_size) runs on the device
    for (int sess = 0; sess < 2; ++sess) {
        LoadedSession& S = sess == 0 ? C : Q;
        int32_t overflow_warnings = 0;
        ck(R.load_session_raw(sess, S.xyzi.data(), S.offsets.data(), S.poses.data(), S.inv_poses.data(), (int)S.keyframe_names.size(), &overflow_warnings),
           sess == 0 ? "load central" : "load query");
        if (overflow_warnings)
            std::fprintf(stderr, "[pcl::VoxelGrid::applyFilter] Leaf size is too small for the input dataset (%d scans returned unchanged)\n", overflow_warnings);
        std::vector<float>().swap(S.xyzi);   // the raw scans now live on the device
    }
    if (compose) {
        int64_t bad = delta_bad.empty() ? 0 : 1;
        if (world > 1) {   // every rank leaves when any rank lacks a delta file
            std::vector<int64_t> all((size_t)world);
            ck(ltr_nccl_allgather_i64(R.ctx, R.nccl_world, &bad, 1, all.data()), "delta file check");
            for (int64_t b : all) bad |= b;
        }
        if (bad) {
            if (delta_bad.empty()) std::fprintf(stderr, "[rank %d] another rank cannot read its delta scans\n", rank);
            return 1;
        }
        ck(R.set_delta_maps(true), "delta maps");
        for (size_t g = 0; g < compose_dirs.size(); ++g)
            ck(R.delta_load(delta_pts[2 * g].data(), delta_off[2 * g].data(), delta_pts[2 * g + 1].data(), delta_off[2 * g + 1].data()), "delta_load");
        std::vector<std::vector<float>>().swap(delta_pts);
        const int T = (int)R.deltas_.size();
        ck(R.compose_changes(0, T), "compose_changes");
        ck(R.rollback(0), "rollback");
        const std::string dc = save_dir + "composed/";
        bool ok = true;
        if (owns_c) {
            for (const char* d : {"scans_pd", "scans_nd_strong", "scans_restored"}) fsmkdir(dc + d);
            ok &= save_scans(R, R.central_sess_.composed_pd_, C.keyframe_names, dc + "scans_pd", false);
            ok &= save_scans(R, R.central_sess_.composed_nd_, C.keyframe_names, dc + "scans_nd_strong", false);
            ok &= save_scans(R, R.central_sess_.keyframe_scans_restored_, C.keyframe_names, dc + "scans_restored", true);
            if (save_map_pcd && rank == 0) ok &= save_cloud(R, R.saved.at("restored_map"), dc + "restored_map.pcd", true);
        }
        if (world > 1 && R.nccl_world >= 0) ltr_nccl_barrier(R.ctx, R.nccl_world);
        if (rank == 0) std::printf(" %d generations composed, outputs written to %s (%s)\n", T, dc.c_str(), ok ? "ok" : "WITH ERRORS");
        return ok ? 0 : 1;
    }
    R.adaptiveThresholdCoeff_ = adaptive_c;   // checked above
    if (adaptive_c != 0.0f && rank == 0)
        std::printf(" Adaptive threshold: coefficient %g, a pixel flags when its diff exceeds fl(%g * scan range) in every remove / revert / ND / PD pass\n",
                    (double)adaptive_c, (double)adaptive_c);
    R.mapBallRadius_ = ball_r;   // checked above
    if (ball_r != 0.0f && rank == 0)
        std::printf(" Map ball: radius %g m, each removeOnce / revertOnce keyframe projects only the map points within it\n", (double)ball_r);
    // one summary line of registrations over both sessions and every rank (a collective: every rank calls it)
    auto icp_summary = [&](const char* what, const IcpStats& a, const IcpStats& b) {
        // [0, kMaxIt] iteration histogram, accepted, keyframes
        constexpr int kMaxIt = 100;
        std::vector<int64_t> h(kMaxIt + 3, 0);
        for (const IcpStats* X : {&a, &b})
            for (size_t k = 0; k < X->iterations.size(); ++k) {
                h[(size_t)std::min(std::max(X->iterations[k], 0), kMaxIt)]++;
                h[kMaxIt + 1] += X->accepted[k];
                h[kMaxIt + 2]++;
            }
        if (world > 1 && R.nccl_world >= 0) {
            std::vector<int64_t> all(h.size() * (size_t)world);
            ck(ltr_nccl_allgather_i64(R.ctx, R.nccl_world, h.data(), (int32_t)h.size(), all.data()), "ICP summary");
            for (size_t j = 0; j < h.size(); ++j) { h[j] = 0; for (int r = 0; r < world; ++r) h[j] += all[(size_t)r * h.size() + j]; }
        }
        int median = 0;
        for (int64_t seen = 0; median <= kMaxIt; ++median) { seen += h[(size_t)median]; if (2 * seen > h[kMaxIt + 2] - 1) break; }
        if (rank == 0)
            std::printf(" %s: %lld of %lld keyframes accepted, median iterations %d\n", what, (long long)h[kMaxIt + 1], (long long)h[kMaxIt + 2],
                        h[kMaxIt + 2] ? median : 0);
    };
    ck(R.run_step0(), "Step 0");
    R.useICPrefinement_ = icp_refinement;
    ck(R.run_step12(), "Step 1-2");
    if (icp_refinement) icp_summary("ICP refinement", R.central_sess_.icp_, R.query_sess_.icp_);
    ck(R.run_step3(), "Step 3");
    if (rank == 0) for (const auto& l : R.log)
        std::printf(" %-18s map %lld  dynamic %lld  -> static %lld  dynamic %lld\n", l.what.c_str(), (long long)l.n_map, (long long)l.n_dynamic,
                    (long long)l.n_static_after, (long long)l.n_dynamic_after);

    // saved maps (all come out of octreeDownsampling: WIDTH 1 / HEIGHT n)
    bool ok = true;
    // a saved map is replicated on the ranks of the group that produced it: its first rank writes it
    const bool group_leader = split ? (rank == 0 || rank == world / 2) : rank == 0;
    for (const auto& kv : R.saved) {
        if (!group_leader) break;
        if (kv.first.rfind("OriginalNoisy", 0) == 0 && !save_map_pcd) continue;   // kFlagSaveMapPointcloud (Removerter.cpp:228)
        ok &= save_cloud(R, kv.second, save_dir + kv.first + ".pcd", true);
    }
    // saveAllTypeOfScans (Removerter.cpp:1607-1630); only keyframe_scans_updated_ went through octreeDownsampling (Session.cpp:374)
    Session& S = R.central_sess_;
    if (owns_c) {   // per-keyframe scans: the owner of the keyframe writes them, under the input scan's name
        ok &= save_scans(R, S.keyframe_scans_updated_, C.keyframe_names, d_updated, true);
        ok &= save_scans(R, S.keyframe_scans_updated_strong_, C.keyframe_names, d_updated_strong, false);
        ok &= save_scans(R, S.keyframe_scans_pd_, C.keyframe_names, d_pd, false);
        ok &= save_scans(R, S.keyframe_scans_strong_pd_, C.keyframe_names, d_pd_strong, false);
        ok &= save_scans(R, S.keyframe_scans_strong_nd_, C.keyframe_names, d_nd_strong, false);
    }
    if (clean_scans >= 0) {
        for (int sess = 0; sess < 2; ++sess) {
            Session& X = sess == 0 ? R.central_sess_ : R.query_sess_;
            const LoadedSession& L = sess == 0 ? C : Q;
            const std::string name = sess == 0 ? "central" : "query";
            ck(R.scansideRemovalForEachScan(X, X, clean_scans), "scansideRemovalForEachScan");   // (C,C), (Q,Q)
            if (R.owns(X)) {
                const std::string ds = save_dir + "scan_static/" + name, dd = save_dir + "scan_dynamic/" + name;
                fsmkdir(ds);
                fsmkdir(dd);
                ok &= save_scans(R, X.scans_static_, L.keyframe_names, ds, false);
                ok &= save_scans(R, X.scans_dynamic_, L.keyframe_names, dd, false);
            }
            if (save_map_pcd && R.owns(X)) {   // saveMapPointcloudByMergingCleanedScans: collective over the ranks holding the session
                const std::string tag = sess == 0 ? "Central" : "Query";
                CloudOwner ms, md;
                ck(R.mergeAndDownsample(X, X.scans_static_.get(), 0.05f, &ms), "merge static scans");
                ck(R.mergeAndDownsample(X, X.scans_dynamic_.get(), 0.05f, &md), "merge dynamic scans");
                if (group_leader) {
                    ok &= save_cloud(R, ms, save_dir + "map_static/" + tag + "StaticScansMergedMapGlobal.pcd", true);
                    ok &= save_cloud(R, md, save_dir + "map_dynamic/" + tag + "DynamicScansMergedMapGlobal.pcd", true);
                }
            }
        }
    }
    if (clean_between >= 0) {
        // (map, scan) = (C,Q): the query's scans against the central map, scan-level PD; (Q,C): the central's against the query map, ND
        for (int scan_sess = 1; scan_sess >= 0; --scan_sess) {
            Session& X = scan_sess == 0 ? R.central_sess_ : R.query_sess_;
            Session& M = scan_sess == 0 ? R.query_sess_ : R.central_sess_;
            const LoadedSession& L = scan_sess == 0 ? C : Q;
            const std::string name = scan_sess == 0 ? "central_vs_query" : "query_vs_central";
            ck(R.scansideRemovalForEachScan(M, X, clean_between, true), "scansideRemovalForEachScan (fine registration)");
            if (R.owns(X)) {
                const std::string ds = save_dir + "scan_static/" + name, dd = save_dir + "scan_dynamic/" + name;
                fsmkdir(ds);
                fsmkdir(dd);
                ok &= save_scans(R, X.scans_static_, L.keyframe_names, ds, false);
                ok &= save_scans(R, X.scans_dynamic_, L.keyframe_names, dd, false);
            }
        }
        icp_summary("Scan-side registration", R.central_sess_.scanside_icp_, R.query_sess_.scanside_icp_);
    }
    if (world > 1 && R.nccl_world >= 0) ltr_nccl_barrier(R.ctx, R.nccl_world);   // nobody leaves before everybody's files are written
    if (rank == 0) std::printf(" outputs written to %s (%s)\n", save_dir.c_str(), ok ? "ok" : "WITH ERRORS");
    return ok ? 0 : 1;
}
