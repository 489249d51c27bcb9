// Internal context / device-container definitions shared by the translation units of libltr_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>   // header-only; a no-op unless a profiler (nsys, ncu --nvtx) is attached
#include <stdint.h>
#include <string>
#include <vector>
#include <cstdio>
#include <map>
#include <chrono>
#include "../../include/ltr_b200.h"
#include "handle_owner.h"

namespace ltr {

struct DevCloud {
    float* base = nullptr;      // one allocation: x | y | z | i, each `cap` floats (cap multiple of 64 -> 256 B aligned components)
    int64_t n = 0, cap = 0;
    uint8_t* flags = nullptr;   // per-point dynamic flags of the last remove pass (lazily allocated, cap bytes)
    bool used = false;
    bool borrowed = false;      // a view into another cloud's storage (ltr_cloud_slice): releasing it frees nothing
    __host__ __device__ float* x() const { return base; }
    __host__ __device__ float* y() const { return base + cap; }
    __host__ __device__ float* z() const { return base + 2 * cap; }
    __host__ __device__ float* i() const { return base + 3 * cap; }
};

struct DevScanSet {
    DevCloud pts;                  // all keyframes back to back
    std::vector<int64_t> h_off;    // K+1 host offsets
    int64_t* d_off = nullptr;      // K+1 device offsets
    int K = 0;
    bool used = false;
    uint64_t serial = 0;           // ltr_ctx::next_serial at creation; the points are written only by the call that creates the set
};

// 24 doubles per keyframe: inverse pose rows 0..2 (12) then pose rows 0..2 (12), row-major 3x4
struct DevPoses {
    double* d = nullptr;
    std::vector<double> h;
    float* d_fast = nullptr;       // K x 16 floats (KfFast, project_fast.cuh)
    std::vector<float> h_fast;
    int K = 0;
    bool used = false;
    uint64_t serial = 0;           // as DevScanSet::serial
};

// Scan-side images of ltr_remove_pass for the keyframes [kf_begin, kf_end) of one scan set (project.cu, scan_images_get), kept between
// passes: they depend on the scans and the image shape, never on the map.  Matched on the serials of the scan set and the poses, which are
// never reused, so a set can never be served for a freed handle whose slot was handed out again.  Each of the context's kMaxScanImageSets
// slots owns one storage block that outlives the sets it holds (dropping a set only marks the slot empty), so the step's passes reuse
// two blocks instead of allocating and freeing multi-GB images.
constexpr int kMaxScanImageSets = 2;   // remove(r), revert(0.95 r), remove(r) alternate between two resolutions
struct ScanImageKey {
    uint64_t scans_serial = 0, poses_serial = 0;
    int kf_begin = 0, kf_end = 0, rows = 0, cols = 0, order = 0, ext_identity = 0, fast_path = 0;
    float vfov = 0.0f, hfov = 0.0f;
    bool operator==(const ScanImageKey& o) const {
        return scans_serial == o.scans_serial && poses_serial == o.poses_serial && kf_begin == o.kf_begin && kf_end == o.kf_end && rows == o.rows &&
               cols == o.cols && order == o.order && ext_identity == o.ext_identity && fast_path == o.fast_path && vfov == o.vfov && hfov == o.hfov;
    }
};
struct ScanImageSet {
    void* block = nullptr;        // storage: rimg | timg | pyr
    size_t cap = 0;               // its bytes
    bool valid = false;           // holds the images of `key`
    ScanImageKey key;
    uint32_t* rimg = nullptr;     // scan range images, (kf_end - kf_begin) x rows x cols
    float* pyr = nullptr;         // sliding-window maxima of tile culling (project_cull.cuh), built for pyr_shortcut
    uint32_t* timg = nullptr;     // test image of the scan-minus-map fast path (scan_test_image_kernel), built for timg_shortcut and the
                                  // threshold coefficient with the bits timg_coeff_bits (0: the constant threshold)
    int pyr_shortcut = -1, timg_shortcut = -1;
    uint32_t timg_coeff_bits = 0;
    uint64_t last_use = 0;
};

struct PtrView { const float *x, *y, *z, *i; int64_t n; };

// one NCCL communicator of a context (nccl_comm.cu)
struct NcclComm {
    void* comm = nullptr;       // ncclComm_t
    int rank = 0, world = 1;
    bool used = false;
    int64_t* h_cnt = nullptr;   // pinned scratch for size exchanges
    int64_t* d_cnt = nullptr;   // device scratch for size exchanges
};

}  // namespace ltr

struct ltr_ctx {
    ltr_config cfg;
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_timer0 = nullptr, ev_timer1 = nullptr;
    std::string err;
    std::vector<ltr::DevCloud> clouds;
    std::vector<ltr::DevScanSet> scansets;
    std::vector<ltr::DevPoses> poses;
    std::vector<ltr::NcclComm> nccl;           // communicators created by ltr_nccl_init / ltr_nccl_split
    int64_t launches = 0;
    uint64_t next_serial = 0;                  // DevScanSet / DevPoses serials
    ltr::ScanImageSet scan_images[ltr::kMaxScanImageSets];   // the least recently used one is refilled first
    uint64_t scan_images_tick = 0;
    int scan_images_busy = 0;                  // a pass is reading a set: the allocator must not free their storage
    bool rs_attr_set = false;    // radix-sort scatter kernel opted in to > 48 KB shared memory on this device
    int64_t vox_shortcuts = 0;   // voxelisations answered by the already-one-point-per-voxel shortcut (util.cu)
    int64_t scanside_stats[4] = {0, 0, 0, 0};   // ltr_scanside_stats (scanside.cu)
    bool ext_identity = true;     // base2lidar/lidar2base exactly identity -> second transform step is exact and skipped
    double* d_ext = nullptr;      // 24 doubles: base2lidar rows 0..2, lidar2base rows 0..2
    double stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    bool stats_counters_pending = false;       // d_counters of the last pass not yet folded into stats[]
    unsigned long long* d_counters = nullptr;  // 4 device counters for pass statistics
    // per-kernel profile of the dominant kernel (map projection): CUDA-event time, launches, algorithmic bytes
    std::vector<cudaEvent_t> ev_pool;          // pairs
    int ev_used = 0;
    double prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // caching device allocator (single stream => a freed block can be handed out again immediately, stream-ordered)
    std::multimap<size_t, void*> free_blocks;  // size -> block
    std::map<void*, size_t> live_blocks;       // block -> size
    size_t cached_bytes = 0, live_bytes = 0, peak_live_bytes = 0;
    size_t cache_limit_bytes = (size_t)48 << 30;
    long n_cuda_malloc = 0, n_cache_hits = 0, n_purges = 0;
    bool trace = false;                        // LTR_TRACE=1: per-entry-point synchronised host timings, dumped at ltr_destroy
    std::map<std::string, std::pair<double, long>> trace_acc; // [0] remove-pass map kernel us, [1] launches, [2] algorithmic bytes, [3] point-projections
                                               // [4] parse map kernel us, [5] launches, [6] algorithmic bytes, [7] point-projections
};

namespace ltr {

extern thread_local std::string g_create_err;

int fail(ltr_ctx* ctx, int code, const char* fmt, ...);

#define LTR_CUDA(ctx, call)                                                                          \
    do {                                                                                             \
        cudaError_t e__ = (call);                                                                    \
        if (e__ != cudaSuccess) return ::ltr::fail(ctx, LTR_ERR_CUDA, "%s failed: %s (%s:%d)", #call, \
                                                   cudaGetErrorString(e__), __FILE__, __LINE__);     \
    } while (0)

#define LTR_TRY(expr)                  \
    do {                               \
        int rc__ = (expr);             \
        if (rc__ != LTR_OK) return rc__; \
    } while (0)

#define LTR_LAUNCH_CHECK(ctx)                                                                         \
    do {                                                                                              \
        (ctx)->launches++;                                                                            \
        cudaError_t e__ = cudaGetLastError();                                                         \
        if (e__ != cudaSuccess) return ::ltr::fail(ctx, LTR_ERR_CUDA, "kernel launch failed: %s (%s:%d)", \
                                                   cudaGetErrorString(e__), __FILE__, __LINE__);      \
    } while (0)

// Entry-point guard: opens an NVTX range, makes the context's GPU the calling thread's current device for the duration of the call (the caller may have
// switched devices -- torch.cuda.set_device, a second context on another GPU -- and cudaMalloc / kernel launches follow the CURRENT
// device) and restores the previous one afterwards; with LTR_TRACE=1 it also times the call on the host between two stream
// synchronisations.
struct ApiTrace {
    ltr_ctx* c; const char* name; double t0; int prev_dev = -1;
    static double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
    ApiTrace(ltr_ctx* ctx, const char* n) : c(ctx), name(n), t0(0) {
        nvtxRangePushA(n);            // every C-ABI entry point is an NVTX range named after itself
        if (!c) return;
        int cur = -1;
        if (cudaGetDevice(&cur) == cudaSuccess && cur != c->device) { prev_dev = cur; cudaSetDevice(c->device); }
        if (c->trace) { cudaStreamSynchronize(c->stream); t0 = now(); }
    }
    ~ApiTrace() {
        nvtxRangePop();
        if (!c) return;
        if (c->trace) { cudaStreamSynchronize(c->stream); auto& a = c->trace_acc[name]; a.first += now() - t0; a.second += 1; }
        if (prev_dev >= 0) cudaSetDevice(prev_dev);
    }
};

// allocation helpers (stream-ordered)
int dev_alloc(ltr_ctx* ctx, void** p, size_t bytes);
void dev_free(ltr_ctx* ctx, void* p);
// Returns a scratch block to the context's cache on every exit path (LTR_TRY / LTR_CUDA return early on errors).
// Declare it right after the pointer it watches; release() frees now (so the block can be reused by the next allocation).
struct ScratchGuard {
    ltr_ctx* ctx;
    void** pp;
    ScratchGuard(ltr_ctx* c, void** p) : ctx(c), pp(p) {}
    ~ScratchGuard() { release(); }
    void release() { if (*pp) { dev_free(ctx, *pp); *pp = nullptr; } }
    ScratchGuard(const ScratchGuard&) = delete;
    ScratchGuard& operator=(const ScratchGuard&) = delete;
};

int cloud_new(ltr_ctx* ctx, int64_t n, CloudOwner* out);         // uninitialised cloud of n points
int cloud_get(ltr_ctx* ctx, ltr_cloud h, DevCloud** c);
int scanset_new(ltr_ctx* ctx, const std::vector<int64_t>& off, ScanSetOwner* out);  // allocates points + uploads offsets
int scanset_get(ltr_ctx* ctx, ltr_scanset h, DevScanSet** s);
int poses_get(ltr_ctx* ctx, ltr_poses h, DevPoses** p);
int cloud_ensure_flags(ltr_ctx* ctx, DevCloud* c);

inline int64_t round_cap(int64_t n) { return ((n > 0 ? n : 1) + 63) / 64 * 64; }
inline PtrView view(const DevCloud& c) { return PtrView{c.x(), c.y(), c.z(), c.i(), c.n}; }

// implemented in util.cu
int stable_partition_by_flag(ltr_ctx* ctx, const DevCloud& in, const uint8_t* flags, int64_t* n_flagged,
                             DevCloud* out_unflagged, DevCloud* out_flagged);   // outputs must be pre-allocated with cap >= in.n
int count_flags(ltr_ctx* ctx, const uint8_t* flags, int64_t n, int64_t* count);
int exclusive_scan_u32(ltr_ctx* ctx, const uint32_t* in, uint32_t* out, int64_t n);  // out[n] elements; returns via out
// *nonfinite (if non-null): number of points with a non-finite x, y or z (NaN coordinates do not show in mn / mx)
int minmax_xyz(ltr_ctx* ctx, const DevCloud& c, float mn[3], float mx[3], uint32_t* nonfinite = nullptr);
// minmax_xyz of a cloud a grid is built over: a point with a non-finite coordinate fails with LTR_ERR_UNSUPPORTED,
// "non-finite <what> coordinates (<count> points<where>)"
int finite_extent(ltr_ctx* ctx, const DevCloud& c, const char* what, float mn[3], float mx[3], const char* where = "");
// pose_offset + [0, scans.K) must be keyframes of poses: LTR_ERR_INVALID otherwise
int check_pose_range(ltr_ctx* ctx, const DevScanSet& scans, const DevPoses& poses, int32_t pose_offset);
// out[j] = off[kf0 + j] - off[kf0] for j <= nkf (device offsets of the keyframes [kf0, kf0 + nkf) relative to the first)
int relative_offsets(ltr_ctx* ctx, const int64_t* off, int kf0, int nkf, int64_t* out);
// stable LSD radix sort of (keys0, vals0) on the key bits [bit_lo, bit_hi), 8 bits per pass, ping-ponging with (keys1, vals1);
// *keys_sorted / *vals_sorted point at whichever buffer holds the result.  vals0 == vals1 == nullptr: keys only.
int radix_sort_pairs(ltr_ctx* ctx, uint64_t* keys0, uint64_t* keys1, uint32_t* vals0, uint32_t* vals1, int64_t n, int bit_lo, int bit_hi,
                     uint64_t** keys_sorted, uint32_t** vals_sorted);
// implemented in nccl_comm.cu (internal helpers of the distributed voxeliser in util.cu)
int nccl_comm_info(ltr_ctx* ctx, int comm, int* rank, int* world);
int nccl_allreduce_u32(ltr_ctx* ctx, int comm, uint32_t* dev, size_t count, int op /* 0 sum, 1 min, 2 max */);
// `send` holds this rank's points grouped by destination rank (segment d has scount[d] points, segments back to back); *recv_out
// receives, in source-rank order, what every rank sent to this one
int nccl_alltoallv_cloud(ltr_ctx* ctx, int comm, const DevCloud& send, const std::vector<int64_t>& scount, CloudOwner* recv_out);

// drops the held scan-image sets (all, or those built from the scan set / poses with that serial); free_storage also returns the slots'
// storage blocks to the allocator (project.cu)
void scan_images_release(ltr_ctx* ctx, uint64_t serial, bool free_storage);
bool scan_images_have_storage(const ltr_ctx* ctx);

int segment_counts(ltr_ctx* ctx, const uint8_t* flags, const DevScanSet& s, std::vector<int64_t>* counts);
int split_scanset_by_flag(ltr_ctx* ctx, const DevScanSet& in, const uint8_t* flags, ltr_scanset* out_unflagged, ltr_scanset* out_flagged);

// The points [base, base + n) of `scans` in the global frame (scan_to_global, ref_math.cuh), written to o*[i - base]; keyframe k's pose
// rows are poses + 24 k + 12, ext is the extrinsic applied first (null: the identity).  oi (optional) receives the intensity.  With the
// device tables T16 / accept (K x 16 floats, K bytes; null: none) the points of keyframe k are then moved by refine_point.
int scans_to_global(ltr_ctx* ctx, const DevScanSet& scans, int64_t base, int64_t n, const double* poses, const double* ext, float* ox,
                    float* oy, float* oz, float* oi, const float* T16 = nullptr, const uint8_t* accept = nullptr);
// The host tables of a refined split (K transforms of 16 floats, K accept flags) to the device: dT (K x 64 B) and dacc (K bytes, 0 / 1).
int upload_refinement(ltr_ctx* ctx, int K, const float* T16, const uint8_t* accepted, float* dT, uint8_t* dacc);

// The end of a scan-set split (ltr_knn_diff, ltr_scanside_split).  The caller sets flags[i] (1: second part) for every point and hands
// over the points' global coordinates, all at once or a keyframe range at a time; relocalise() moves them back to their keyframes'
// frames (global2local, Session.cpp:603-604: the inverse pose at poses + 24 k, then base2lidar) into a copy of the scans that keeps
// their intensity, and finish() splits that copy by the flags, order preserved, or gives K empty keyframes when the set has no points.
// The copy is allocated by the first relocalise(), so a caller that frees its search structures first never holds both.
class ScanSplit {
public:
    uint8_t* flags = nullptr;   // one byte per point, after init()
    ScanSplit(ltr_ctx* ctx, const DevScanSet& scans, const double* poses) : ctx_(ctx), scans_(scans), poses_(poses), reloc_(ctx) {}
    ~ScanSplit() { if (flags) dev_free(ctx_, flags); }
    int init();
    int relocalise(int64_t base, int64_t n, const float* gx, const float* gy, const float* gz);
    int finish(ltr_scanset* out0, ltr_scanset* out1);
    ScanSplit(const ScanSplit&) = delete;
    ScanSplit& operator=(const ScanSplit&) = delete;
private:
    ltr_ctx* ctx_;
    DevScanSet scans_;
    const double* poses_;
    CloudOwner reloc_;
};

// A launch-size knob: the environment variable `name` clamped to [1, hi], or def when it is unset or empty.
int64_t env_points(const char* name, int64_t def, int64_t hi);
// Cuts the keyframes of the offsets off[0..K] into launches [cut[j], cut[j + 1]) of at most max_kf keyframes and at most cap points,
// except that a keyframe is never split (a larger one goes alone); *max_points = the largest launch's points.
std::vector<int> plan_keyframe_chunks(const std::vector<int64_t>& off, int64_t cap, int max_kf, int64_t* max_points);

constexpr int kKnnMaxK = 16;   // the largest k of every kNN search

// The thresholded kNN decision of the kNN diff and ltr_knn_split_cloud (knn.cu) against one target, built once and applied to any number
// of query views already in the target's frame (also scan-side removal, scanside.cu): a dense grid (origin, inv_cell, dim; cell_start has
// one entry per cell plus one, sorted holds the points cell by cell).  knn_target_build: 1 <= k <= kKnnMaxK, thr > 0, target of >= 1
// points, finite unless it has fewer than k; the caller returns *block to the allocator.  knn_target_label: label[i] = 1 if |avg| >= thr
// ("far"), else 0.
struct KnnTarget {
    double origin[3] = {0, 0, 0};
    double inv_cell = 0;
    int dim[3] = {0, 0, 0};
    const uint32_t* cell_start = nullptr;
    const float4* sorted = nullptr;
    PtrView small{nullptr, nullptr, nullptr, nullptr, 0};   // targets of fewer than k points are searched by brute force
};
int knn_target_build(ltr_ctx* ctx, const DevCloud& target, int k, float thr, KnnTarget* t, void** block);
int knn_target_label(ltr_ctx* ctx, const KnnTarget& t, PtrView q, int k, float thr, uint8_t* label);

// ltr_knn_diff (T16 = accepted = null) and ltr_knn_diff_refined (knn.cu): with T16 the global points of keyframe k with accepted[k] != 0
// are moved by T16 + 16 k before they are labelled.  refined: K > 0 keyframes without T16 or accepted are LTR_ERR_INVALID.
int knn_diff(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud target_h, int32_t k, float thr, bool refined,
             const float* T16, const uint8_t* accepted, ltr_scanset* out_coexist, ltr_scanset* out_diff);

}  // namespace ltr
