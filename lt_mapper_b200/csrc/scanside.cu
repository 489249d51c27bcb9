// libltr_b200.so -- scan-side removal: every keyframe's own scan, at full resolution, split into static and dynamic points.
//
// Reference functions (kept in the node's sources but commented out; params_ltmapper.yaml's saveCleanScansPCD asks for their output):
//   Removerter::removeDynamicPointsOfScanByKnn(int, const Session&, kdtree)   ltremovert/src/Removerter.cpp:1019-1069   criterion "map"
//   Removerter::removeDynamicPointsOfScanByKnn(int)                             ltremovert/src/Removerter.cpp:1071-1123   "scan minus map"
//   Removerter::scansideRemovalForEachScan(map_sess, scan_sess)                 ltremovert/src/Removerter.cpp:1253-1310
// Transforms: scan_global = local2global(scan, pose, kSE3MatExtrinsicLiDARtoPoseBase), the live 3-argument overload of
// utility.cpp:160-168 (the commented code calls a 2-argument overload that no longer exists; partitionLowDynamicPointsOfScanByKnn passes
// the other extrinsic; with the identity extrinsic all of them agree); both parts go back with global2local(..., inv_pose,
// kSE3MatExtrinsicPoseBasetoLiDAR) (utility.cpp:194-202).
//
// "map" needs only the decision |avg_map| < thr: that is knn.cu's bounded 27-cell grid search (its header has the proof).
// "scan minus map" needs the exact VALUES of avg_scan and avg_map -- two large averages can differ by less than thr -- so no radius bound
// applies.  Both averages come from an exact k-NN over the sparse grid levels of sparse_grid.cuh (segment = keyframe of the launch for
// the own-scan targets, 0 for the map): a query searches shell by shell and stops after shell s when the block holds every cell, or when
// its k-th smallest computed distance D_k satisfies D_k <= ((s - 2^-6) c)^2 (1 - 2^-20), or D_k = 0.  sparse_grid.cuh's header proves
// the stop exact.
// Two passes: a bounded pass on the finest level (c0 = 0.25 m, shells 0..2) settles almost every point.  The rest (isolated returns at
// long range, queries far from the map) are compacted into a list and searched on levels of 4x, 16x, ... the cell side, bounded again
// except on the coarsest level (at most 10 cells per axis), which searches until the stop rule holds.  A level changes the cost only.
// Memory: keyframes go through in launches of at most LTR_SCANSIDE_CHUNK_POINTS points (default 2^24, a keyframe is never split); per
// launch the global coordinates (16 B/point), two averages (8 B/point), two unsettled lists (8 B/point) and one own-scan grid level
// (28 B/point, plus 32 B/point of sort scratch while it is built).  The map's levels (28 B per map point each) are built once per call and
// only as far as some query needs them.  Beside that the call holds one flag byte per point and a relocalised copy of the scans
// (16 B/point) for the final order-preserving compaction, as ltr_knn_diff does.  All of it comes from the context's caching allocator and
// is returned before the call ends.
// ltr_scanside_split_refined (the fine registration between sessions, Removerter.cpp:950-1017; DESIGN.md §5.4) is the same body with a
// per-keyframe transform table on the device (64 B + 1 B per keyframe), applied in the chunk's global-coordinate step.
#include "ltr_internal.cuh"
#include "ref_math.cuh"
#include "device_util.cuh"
#include "sparse_grid.cuh"
#include <algorithm>
#include <cmath>

namespace ltr {

namespace {

constexpr int kSegShift = kGridSegShift;
constexpr int kMaxSegments = kGridMaxSegments;   // 8192 keyframes per launch
constexpr int kBoundedShells = 2;
constexpr int64_t kChunkPoints = (int64_t)1 << 24;

// ---- level build -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) level_key_kernel(PtrView p, const int64_t* __restrict__ off, int nseg, Level L,
                                                        unsigned long long* __restrict__ keys, uint32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int seg = off ? find_kf(off, nseg, i) : 0;
    long long c[3];
    const float v[3] = {p.x[i], p.y[i], p.z[i]};
#pragma unroll
    for (int d = 0; d < 3; ++d) c[d] = min(max(cell_index((double)v[d], L.origin[d], L.inv_cell), 0ll), (long long)L.dim[d] - 1);
    keys[i] = cell_key(seg, c[0], c[1], c[2]);
    idx[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) level_head_kernel(const unsigned long long* __restrict__ keys, int64_t n, uint32_t* __restrict__ head) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}

__global__ void __launch_bounds__(256) level_compact_kernel(PtrView p, const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ idx,
                                                            const uint32_t* __restrict__ head, const uint32_t* __restrict__ pos, int64_t n,
                                                            unsigned long long* __restrict__ ukeys, uint32_t* __restrict__ start,
                                                            float4* __restrict__ pts, uint32_t* __restrict__ ncell) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (head[i]) { ukeys[pos[i]] = keys[i]; start[pos[i]] = (uint32_t)i; }
    if (i == n - 1) { const uint32_t m = pos[i] + head[i]; start[m] = (uint32_t)n; *ncell = m; }
    const uint32_t j = idx[i];
    pts[i] = make_float4(p.x[j], p.y[j], p.z[j], __uint_as_float(j));
}

__global__ void level_segments_kernel(const unsigned long long* __restrict__ ukeys, const uint32_t* __restrict__ ncell, int nseg,
                                      uint32_t* __restrict__ seg_first) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s > nseg) return;
    const unsigned long long key = (unsigned long long)s << kSegShift;
    uint32_t lo = 0, hi = *ncell;
    if (s < nseg) {
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (ukeys[mid] < key) lo = mid + 1; else hi = mid; }
    } else lo = hi;
    seg_first[s] = lo;
}

}  // namespace

// sparse_grid.cuh
int build_level(ltr_ctx* ctx, PtrView p, const int64_t* d_off, int nseg, const float mn[3], const float mx[3], double cell, bool final_level,
                LevelBuf* out) {
    Level L{};
    L.inv_cell = 1.0 / cell;
    L.cell = 1.0 / L.inv_cell;
    for (int d = 0; d < 3; ++d) {
        L.origin[d] = (double)mn[d] - cell;   // one guard cell below the minimum
        L.dim[d] = (int)std::floor(((double)mx[d] - L.origin[d]) * L.inv_cell) + 2;
    }
    L.final_level = final_level ? 1 : 0;
    const int64_t n = p.n;
    auto pad = [](size_t b) { return (b + 255) / 256 * 256; };
    const size_t b_keys = pad((size_t)n * 8), b_start = pad((size_t)(n + 1) * 4), b_pts = pad((size_t)n * 16), b_seg = pad((size_t)(nseg + 2) * 4);
    void* blk = nullptr;
    ScratchGuard g_blk(ctx, &blk);
    LTR_TRY(dev_alloc(ctx, &blk, b_keys + b_start + b_pts + b_seg));
    char* c = (char*)blk;
    unsigned long long* ukeys = (unsigned long long*)c;
    uint32_t* start = (uint32_t*)(c + b_keys);
    float4* pts = (float4*)(c + b_keys + b_start);
    uint32_t* seg_first = (uint32_t*)(c + b_keys + b_start + b_pts);
    uint32_t* ncell = seg_first + nseg + 1;
    void* tmp = nullptr;
    ScratchGuard g_tmp(ctx, &tmp);
    const size_t b_k = pad((size_t)n * 8), b_v = pad((size_t)n * 4);
    LTR_TRY(dev_alloc(ctx, &tmp, 2 * b_k + 4 * b_v));
    char* t = (char*)tmp;
    unsigned long long* k0 = (unsigned long long*)t;
    unsigned long long* k1 = (unsigned long long*)(t + b_k);
    uint32_t* v0 = (uint32_t*)(t + 2 * b_k);
    uint32_t* v1 = (uint32_t*)(t + 2 * b_k + b_v);
    uint32_t* head = (uint32_t*)(t + 2 * b_k + 2 * b_v);
    uint32_t* pos = (uint32_t*)(t + 2 * b_k + 3 * b_v);
    const unsigned nb = (unsigned)((n + 255) / 256);
    level_key_kernel<<<nb, 256, 0, ctx->stream>>>(p, d_off, nseg, L, k0, v0);
    LTR_LAUNCH_CHECK(ctx);
    int seg_bits = 0;
    while ((1 << seg_bits) < nseg) ++seg_bits;
    uint64_t* ks;
    uint32_t* vs;
    LTR_TRY(radix_sort_pairs(ctx, (uint64_t*)k0, (uint64_t*)k1, v0, v1, n, 0, kSegShift + seg_bits, &ks, &vs));
    level_head_kernel<<<nb, 256, 0, ctx->stream>>>((const unsigned long long*)ks, n, head);
    LTR_LAUNCH_CHECK(ctx);
    LTR_TRY(exclusive_scan_u32(ctx, head, pos, n));
    level_compact_kernel<<<nb, 256, 0, ctx->stream>>>(p, (const unsigned long long*)ks, vs, head, pos, n, ukeys, start, pts, ncell);
    LTR_LAUNCH_CHECK(ctx);
    level_segments_kernel<<<(nseg + 1 + 127) / 128, 128, 0, ctx->stream>>>(ukeys, ncell, nseg, seg_first);
    LTR_LAUNCH_CHECK(ctx);
    g_tmp.release();
    L.keys = ukeys; L.start = start; L.pts = pts; L.seg_first = seg_first;
    out->L = L;
    out->block = blk;
    blk = nullptr;   // ownership moves to out
    return LTR_OK;
}

namespace {

// ---- exact k-NN ----------------------------------------------------------------------------------------------------------------------
// the K smallest computed distances with the shell search's stop rule for them (sparse_grid.cuh's header)
template <int K>
struct Best : TopK<K> {
    __device__ __forceinline__ void push(float v, const float4&) { TopK<K>::push(v); }
    __device__ __forceinline__ bool settled(long long s, double cell) const {
        if (!this->has(K)) return false;
        const double dk = (double)this->d[K - 1], b = shell_bound(s, cell);
        return dk == 0.0 || (s > 0 && dk <= b);
    }
};

// Exact mean of the k smallest squared distances from q to the points of segment `seg`.  false: not settled within max_shell shells on a
// bounded level.
template <int K>
__device__ bool knn_exact_avg(const Level& L, int seg, float qx, float qy, float qz, int max_shell, float* avg) {
    Best<K> b;
    b.init();
    if (!shell_search(L, seg, qx, qy, qz, max_shell, b)) return false;
    *avg = b.mean(K);
    return true;
}

// One level for the queries list[0..n) (list == nullptr: the queries 0..n): settled ones write avg[i], the others go to next.
template <int K>
__global__ void __launch_bounds__(128) exact_knn_kernel(Level L, PtrView q, const int64_t* __restrict__ q_off, int nseg,
                                                        const uint32_t* __restrict__ list, int64_t n, int max_shell, float* __restrict__ avg,
                                                        uint32_t* __restrict__ next, unsigned int* __restrict__ next_cnt) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t i = list ? list[t] : (uint32_t)t;
    const int seg = q_off ? find_kf(q_off, nseg, i) : 0;
    float a;
    if (knn_exact_avg<K>(L, seg, q.x[i], q.y[i], q.z[i], max_shell, &a)) avg[i] = a;
    else next[atomicAdd(next_cnt, 1u)] = i;
}

int launch_exact_knn(ltr_ctx* ctx, int k, const Level& L, PtrView q, const int64_t* q_off, int nseg, const uint32_t* list, int64_t n,
                     float* avg, uint32_t* next, unsigned int* next_cnt) {
    if (n == 0) return LTR_OK;
    const unsigned nb = (unsigned)((n + 127) / 128);
    switch (k) {
#define LTR_SCANSIDE_CASE(KK) \
        case KK: exact_knn_kernel<KK><<<nb, 128, 0, ctx->stream>>>(L, q, q_off, nseg, list, n, kBoundedShells, avg, next, next_cnt); break;
        LTR_SCANSIDE_CASE(1) LTR_SCANSIDE_CASE(2) LTR_SCANSIDE_CASE(3) LTR_SCANSIDE_CASE(4) LTR_SCANSIDE_CASE(5) LTR_SCANSIDE_CASE(6)
        LTR_SCANSIDE_CASE(7) LTR_SCANSIDE_CASE(8) LTR_SCANSIDE_CASE(9) LTR_SCANSIDE_CASE(10) LTR_SCANSIDE_CASE(11) LTR_SCANSIDE_CASE(12)
        LTR_SCANSIDE_CASE(13) LTR_SCANSIDE_CASE(14) LTR_SCANSIDE_CASE(15) LTR_SCANSIDE_CASE(16)
#undef LTR_SCANSIDE_CASE
        default: return fail(ctx, LTR_ERR_UNSUPPORTED, "k = %d outside [1, %d]", k, kKnnMaxK);
    }
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

// avg[i] for every query of q against the target pyramid; *unsettled = queries the bounded pass on the finest level left over.
int exact_avg_all(ltr_ctx* ctx, Pyramid& T, int k, PtrView q, const int64_t* q_off, int nseg, float* avg, uint32_t* list_a,
                  uint32_t* list_b, unsigned int* d_cnt, int64_t* unsettled) {
    const uint32_t* list = nullptr;
    int64_t n = q.n;
    *unsettled = 0;
    for (int l = 0; n > 0; ++l) {
        const Level* L;
        LTR_TRY(T.get(l, &L));
        uint32_t* next = (list == list_a) ? list_b : list_a;
        LTR_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, sizeof(unsigned int), ctx->stream));
        LTR_TRY(launch_exact_knn(ctx, k, *L, q, q_off, nseg, list, n, avg, next, d_cnt));
        if (L->final_level) break;
        unsigned int h = 0;
        LTR_CUDA(ctx, cudaMemcpyAsync(&h, d_cnt, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (l == 0) *unsettled = h;
        list = next;
        n = h;
    }
    return LTR_OK;
}

// ---- decisions -----------------------------------------------------------------------------------------------------------------------
// fabsf(avg_scan - avg_map) < thr -> static (Removerter.cpp:1107), the subtraction in f32
__global__ void __launch_bounds__(256) scanside_diff_kernel(const float* __restrict__ avg_scan, const float* __restrict__ avg_map, int64_t n,
                                                            float thr, uint8_t* __restrict__ flag) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    flag[t] = (fabsf(fs(avg_scan[t], avg_map[t])) < thr) ? 0 : 1;
}

// ltr_scanside_split (refined = false, T16 = accepted = null) and ltr_scanside_split_refined: with refined, the global points of keyframe
// k with accepted[k] != 0 are moved by T16 + 16 k in the chunk's global-coordinate step, before the finite check, both searches and the
// relocalisation; K > 0 keyframes without T16 or accepted are LTR_ERR_INVALID.
int scanside_split(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud map_h, int32_t criterion, int32_t k,
                   float thr, bool refined, const float* T16, const uint8_t* accepted, ltr_scanset* out_static, ltr_scanset* out_dynamic) {
    DevScanSet* sp;
    DevPoses* pp;
    DevCloud* mp;
    LTR_TRY(scanset_get(ctx, scans_h, &sp));
    LTR_TRY(poses_get(ctx, poses_h, &pp));
    LTR_TRY(cloud_get(ctx, map_h, &mp));
    if (criterion != LTR_SCANSIDE_MAP && criterion != LTR_SCANSIDE_SCAN_MINUS_MAP) return fail(ctx, LTR_ERR_INVALID, "unknown criterion %d", criterion);
    if (k < 1 || k > kKnnMaxK) return fail(ctx, LTR_ERR_UNSUPPORTED, "k = %d outside [1, %d]", k, kKnnMaxK);
    if (!(thr > 0.0f)) return fail(ctx, LTR_ERR_INVALID, "threshold must be positive");
    LTR_TRY(check_pose_range(ctx, *sp, *pp, pose_offset));
    if (mp->n < 1) return fail(ctx, LTR_ERR_UNSUPPORTED, "empty map (PCL's nearestKSearch asserts on an empty tree)");
    if (refined && sp->K > 0 && (!T16 || !accepted)) return fail(ctx, LTR_ERR_INVALID, "null transforms or accept mask");
    const DevScanSet scans = *sp;
    const DevPoses poses = *pp;
    const DevCloud map = *mp;
    for (int j = 0; j < 4; ++j) ctx->scanside_stats[j] = 0;
    ctx->scanside_stats[0] = scans.pts.n;
    float map_mn[3], map_mx[3];
    LTR_TRY(finite_extent(ctx, map, "map", map_mn, map_mx));
    const int64_t n = scans.pts.n;
    const double* pose0 = poses.d + (size_t)pose_offset * 24;
    ScanSplit split(ctx, scans, pose0);
    LTR_TRY(split.init());
    if (n > 0) {
        int64_t max_chunk = 0;
        const std::vector<int> kf_cut = plan_keyframe_chunks(scans.h_off, env_points("LTR_SCANSIDE_CHUNK_POINTS", kChunkPoints, (int64_t)1 << 30),
                                                             kMaxSegments, &max_chunk);
        if (max_chunk >= ((int64_t)1 << 32)) return fail(ctx, LTR_ERR_UNSUPPORTED, "a keyframe of %lld points", (long long)max_chunk);
        const int64_t ccap = round_cap(max_chunk);
        void* work = nullptr;
        ScratchGuard g_work(ctx, &work);
        // chunk global coordinates (a DevCloud layout, for minmax_xyz) | avg_map | avg_scan | two lists | counter | chunk offsets |
        // refinement transforms | accept flags
        const size_t b_g = (size_t)ccap * 16, b_f = (size_t)ccap * 4, b_off = ((size_t)kMaxSegments + 1) * 8;
        const size_t b_T = refined ? ((size_t)scans.K * 64 + 255) / 256 * 256 : 0, b_acc = refined ? (size_t)scans.K : 0;
        LTR_TRY(dev_alloc(ctx, &work, b_g + 4 * b_f + 256 + b_off + b_T + b_acc));
        float* dT = nullptr;
        uint8_t* dacc = nullptr;
        if (refined) {
            dT = (float*)((char*)work + b_g + 4 * b_f + 256 + b_off);
            dacc = (uint8_t*)dT + b_T;
            LTR_TRY(upload_refinement(ctx, scans.K, T16, accepted, dT, dacc));
        }
        DevCloud g;
        g.base = (float*)work; g.cap = ccap;
        float* avg_map = (float*)((char*)work + b_g);
        float* avg_scan = avg_map + ccap;
        uint32_t* list_a = (uint32_t*)(avg_scan + ccap);
        uint32_t* list_b = list_a + ccap;
        unsigned int* d_cnt = (unsigned int*)(list_b + ccap);
        int64_t* c_off = (int64_t*)((char*)work + b_g + 4 * b_f + 256);
        KnnTarget kt;
        void* kt_block = nullptr;
        ScratchGuard g_kt(ctx, &kt_block);
        Pyramid mapT(ctx);
        if (criterion == LTR_SCANSIDE_MAP) LTR_TRY(knn_target_build(ctx, map, k, thr, &kt, &kt_block));
        else mapT.init(view(map), nullptr, 1, map_mn, map_mx);
        for (size_t c = 0; c + 1 < kf_cut.size(); ++c) {
            const int kf0 = kf_cut[c], kf1 = kf_cut[c + 1], nkf = kf1 - kf0;
            const int64_t base = scans.h_off[kf0], m = scans.h_off[kf1] - base;
            ctx->scanside_stats[3]++;
            if (m == 0) continue;
            // local2global with lidar2base (file header), then an accepted keyframe's registration
            LTR_TRY(scans_to_global(ctx, scans, base, m, pose0, ctx->ext_identity ? nullptr : ctx->d_ext + 12, g.x(), g.y(), g.z(), nullptr, dT,
                                    dacc));
            g.n = m;
            float mn[3], mx[3];
            char where[48];
            snprintf(where, sizeof(where), " in keyframes [%d,%d)", kf0, kf1);
            LTR_TRY(finite_extent(ctx, g, "scan", mn, mx, where));
            const PtrView q = view(g);
            uint8_t* fl = split.flags + base;
            if (criterion == LTR_SCANSIDE_MAP) {
                // |avg_map| < thr -> static (Removerter.cpp:1056)
                LTR_TRY(knn_target_label(ctx, kt, q, k, thr, fl));
            } else {
                LTR_TRY(relative_offsets(ctx, scans.d_off, kf0, nkf, c_off));
                int64_t un = 0;
                LTR_TRY(exact_avg_all(ctx, mapT, k, q, nullptr, 1, avg_map, list_a, list_b, d_cnt, &un));
                ctx->scanside_stats[1] += un;
                Pyramid self(ctx);
                self.init(q, c_off, nkf, mn, mx);
                LTR_TRY(exact_avg_all(ctx, self, k, q, c_off, nkf, avg_scan, list_a, list_b, d_cnt, &un));
                ctx->scanside_stats[2] += un;
                self.release();
                scanside_diff_kernel<<<(unsigned)((m + 255) / 256), 256, 0, ctx->stream>>>(avg_scan, avg_map, m, thr, fl);
                LTR_LAUNCH_CHECK(ctx);
            }
            LTR_TRY(split.relocalise(base, m, g.x(), g.y(), g.z()));
        }
        mapT.release();
        g_kt.release();
        g_work.release();
    }
    return split.finish(out_static, out_dynamic);
}

}  // namespace
}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_scanside_split(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud map_h, int32_t criterion,
                       int32_t k, float thr, ltr_scanset* out_static, ltr_scanset* out_dynamic) {
    ApiTrace tr__(ctx, "ltr_scanside_split");
    if (!ctx) return LTR_ERR_INVALID;
    return scanside_split(ctx, scans_h, poses_h, pose_offset, map_h, criterion, k, thr, false, nullptr, nullptr, out_static, out_dynamic);
}

int ltr_scanside_split_refined(ltr_ctx* ctx, ltr_scanset scans_h, ltr_poses poses_h, int32_t pose_offset, ltr_cloud map_h, int32_t criterion,
                               int32_t k, float thr, const float* T16, const uint8_t* accepted, ltr_scanset* out_static,
                               ltr_scanset* out_dynamic) {
    ApiTrace tr__(ctx, "ltr_scanside_split_refined");
    if (!ctx) return LTR_ERR_INVALID;
    return scanside_split(ctx, scans_h, poses_h, pose_offset, map_h, criterion, k, thr, true, T16, accepted, out_static, out_dynamic);
}

int ltr_scanside_stats(ltr_ctx* ctx, int64_t* stats4) {
    if (!ctx || !stats4) return LTR_ERR_INVALID;
    for (int j = 0; j < 4; ++j) stats4[j] = ctx->scanside_stats[j];
    return LTR_OK;
}

// The exact k-NN averages of ltr_scanside_split (Pyramid + exact_avg_all, as its "scan minus map" branch calls them) for every point of
// `query_h`, in one launch: against target_h (self == 0, avg_map), or keyframe j against its own points (self != 0, avg_scan).
int ltr_debug_exact_knn_avg(ltr_ctx* ctx, ltr_scanset query_h, ltr_cloud target_h, int32_t self, int32_t k, float* avg_out, int64_t* unsettled) {
    ApiTrace tr__(ctx, "ltr_debug_exact_knn_avg");
    if (!ctx || !avg_out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevScanSet* sp;
    LTR_TRY(scanset_get(ctx, query_h, &sp));
    DevCloud* tp = nullptr;
    if (!self) LTR_TRY(cloud_get(ctx, target_h, &tp));
    if (k < 1 || k > kKnnMaxK) return fail(ctx, LTR_ERR_UNSUPPORTED, "k = %d outside [1, %d]", k, kKnnMaxK);
    if (self && sp->K > kMaxSegments) return fail(ctx, LTR_ERR_UNSUPPORTED, "%d keyframes in one launch (at most %d)", sp->K, kMaxSegments);
    if (!self && tp->n < 1) return fail(ctx, LTR_ERR_UNSUPPORTED, "empty target");
    const DevScanSet q = *sp;
    const int64_t n = q.pts.n;
    if (n >= ((int64_t)1 << 32)) return fail(ctx, LTR_ERR_UNSUPPORTED, "%lld query points", (long long)n);
    float qmn[3], qmx[3];
    if (n > 0) LTR_TRY(finite_extent(ctx, q.pts, "query", qmn, qmx));
    Pyramid T(ctx);
    if (!self) {
        float mn[3], mx[3];
        LTR_TRY(finite_extent(ctx, *tp, "target", mn, mx));
        T.init(view(*tp), nullptr, 1, mn, mx);
    }
    int64_t un = 0;
    if (n > 0) {
        if (self) T.init(view(q.pts), q.d_off, q.K, qmn, qmx);
        const int64_t cap = round_cap(n);
        void* work = nullptr;
        ScratchGuard g_work(ctx, &work);
        LTR_TRY(dev_alloc(ctx, &work, (size_t)cap * 12 + 256));   // avg | two lists | counter
        float* avg = (float*)work;
        uint32_t* list_a = (uint32_t*)(avg + cap);
        uint32_t* list_b = list_a + cap;
        unsigned int* d_cnt = (unsigned int*)(list_b + cap);
        LTR_TRY(exact_avg_all(ctx, T, k, view(q.pts), self ? q.d_off : nullptr, self ? q.K : 1, avg, list_a, list_b, d_cnt, &un));
        LTR_CUDA(ctx, cudaMemcpyAsync(avg_out, avg, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (unsettled) *unsettled = un;
    return LTR_OK;
}

}  // extern "C"
