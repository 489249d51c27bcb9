// libltr_b200.so -- context, handle tables and data movement of the C-ABI (include/ltr_b200.h).
#include "ltr_internal.cuh"
#include <cstdarg>
#include <cstring>
#include <cmath>
#include <cstdlib>

thread_local std::string ltr::g_create_err;

namespace ltr {

int fail(ltr_ctx* ctx, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf; else g_create_err = buf;
    return code;
}

// Caching allocator.  cudaMallocAsync's pool showed multi-millisecond stalls (pool growth / remapping) at unpredictable
// points of a step; every allocation of this library is used on ctx->stream only, so a block freed by the host after the
// kernels using it were enqueued can be re-issued immediately (stream order protects it).  Blocks are rounded to 512 B /
// 2 MiB granules and recycled best-fit (at most 25 % + 2 MiB larger than requested); cudaMalloc only on a miss (warm-up).
static size_t round_block(size_t bytes) {
    if (bytes == 0) bytes = 1;
    const size_t g = bytes >= (1u << 20) ? (size_t)(2u << 20) : (size_t)512;
    return (bytes + g - 1) / g * g;
}
int dev_alloc(ltr_ctx* ctx, void** p, size_t bytes) {
    *p = nullptr;
    const size_t want = round_block(bytes);
    auto it = ctx->free_blocks.lower_bound(want);
    if (it != ctx->free_blocks.end() && it->first <= want + want / 4 + (size_t)(2u << 20)) {
        *p = it->second;
        ctx->live_blocks[*p] = it->first;
        ctx->cached_bytes -= it->first;
        ctx->live_bytes += it->first;
        if (ctx->live_bytes > ctx->peak_live_bytes) ctx->peak_live_bytes = ctx->live_bytes;
        ctx->n_cache_hits++;
        ctx->free_blocks.erase(it);
        return LTR_OK;
    }
    cudaError_t e = cudaMalloc(p, want);
    const bool can_drop_images = scan_images_have_storage(ctx) && !ctx->scan_images_busy;
    if (e == cudaErrorMemoryAllocation && (!ctx->free_blocks.empty() || can_drop_images)) {   // give the cache back and retry once
        cudaGetLastError();
        if (can_drop_images) scan_images_release(ctx, 0, true);   // the scan-image storage of ltr_remove_pass goes first (into the cache, freed below)
        cudaStreamSynchronize(ctx->stream);
        for (auto& kv : ctx->free_blocks) cudaFree(kv.second);
        ctx->free_blocks.clear();
        ctx->cached_bytes = 0;
        e = cudaMalloc(p, want);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(ctx, e == cudaErrorMemoryAllocation ? LTR_ERR_NOMEM : LTR_ERR_CUDA, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    }
    ctx->live_blocks[*p] = want;
    ctx->live_bytes += want;
    if (ctx->live_bytes > ctx->peak_live_bytes) ctx->peak_live_bytes = ctx->live_bytes;
    ctx->n_cuda_malloc++;
    return LTR_OK;
}
void dev_free(ltr_ctx* ctx, void* p) {
    if (!p) return;
    auto it = ctx->live_blocks.find(p);
    if (it == ctx->live_blocks.end()) return;
    const size_t sz = it->second;
    ctx->live_blocks.erase(it);
    ctx->live_bytes -= sz;
    ctx->free_blocks.emplace(sz, p);
    ctx->cached_bytes += sz;
    if (ctx->cached_bytes > ctx->cache_limit_bytes) {   // bound the cache: drop everything that is not in use
        ctx->n_purges++;
        cudaStreamSynchronize(ctx->stream);
        for (auto& kv : ctx->free_blocks) cudaFree(kv.second);
        ctx->free_blocks.clear();
        ctx->cached_bytes = 0;
    }
}

int cloud_new(ltr_ctx* ctx, int64_t n, CloudOwner* out) {
    if (n < 0) return fail(ctx, LTR_ERR_INVALID, "negative cloud size");
    int slot = -1;
    for (size_t i = 0; i < ctx->clouds.size(); ++i) if (!ctx->clouds[i].used) { slot = (int)i; break; }
    if (slot < 0) { ctx->clouds.push_back(DevCloud()); slot = (int)ctx->clouds.size() - 1; }
    DevCloud c;
    c.n = n; c.cap = round_cap(n); c.used = true;
    void* p;
    LTR_TRY(dev_alloc(ctx, &p, (size_t)c.cap * 4 * sizeof(float)));
    c.base = (float*)p;
    ctx->clouds[slot] = c;
    *out = CloudOwner(ctx, slot);
    return LTR_OK;
}
int cloud_get(ltr_ctx* ctx, ltr_cloud h, DevCloud** c) {
    if (h < 0 || h >= (int)ctx->clouds.size() || !ctx->clouds[h].used) return fail(ctx, LTR_ERR_INVALID, "invalid cloud handle %d", h);
    *c = &ctx->clouds[h];
    return LTR_OK;
}
static void cloud_release(ltr_ctx* ctx, DevCloud* c) {
    if (!c->borrowed) dev_free(ctx, c->base);
    dev_free(ctx, c->flags);
    *c = DevCloud();
}
int cloud_ensure_flags(ltr_ctx* ctx, DevCloud* c) {
    if (c->flags) return LTR_OK;
    void* p;
    LTR_TRY(dev_alloc(ctx, &p, (size_t)c->cap));
    c->flags = (uint8_t*)p;
    LTR_CUDA(ctx, cudaMemsetAsync(c->flags, 0, (size_t)c->cap, ctx->stream));
    return LTR_OK;
}
int scanset_new(ltr_ctx* ctx, const std::vector<int64_t>& off, ScanSetOwner* out) {
    const int K = (int)off.size() - 1;
    if (K < 0) return fail(ctx, LTR_ERR_INVALID, "scanset needs K+1 offsets");
    for (int k = 0; k < K; ++k) if (off[k + 1] < off[k]) return fail(ctx, LTR_ERR_INVALID, "scanset offsets must be non-decreasing");
    if (off[0] != 0) return fail(ctx, LTR_ERR_INVALID, "scanset offsets must start at 0");
    int slot = -1;
    for (size_t i = 0; i < ctx->scansets.size(); ++i) if (!ctx->scansets[i].used) { slot = (int)i; break; }
    if (slot < 0) { ctx->scansets.push_back(DevScanSet()); slot = (int)ctx->scansets.size() - 1; }
    DevScanSet s;
    s.K = K; s.h_off = off; s.used = true; s.serial = ++ctx->next_serial;
    s.pts.n = off[K]; s.pts.cap = round_cap(off[K]); s.pts.used = true;
    void *p_pts = nullptr, *p_off = nullptr;
    ScratchGuard g_pts(ctx, &p_pts), g_off(ctx, &p_off);   // disarmed once the handle owns both blocks
    LTR_TRY(dev_alloc(ctx, &p_pts, (size_t)s.pts.cap * 4 * sizeof(float)));
    s.pts.base = (float*)p_pts;
    LTR_TRY(dev_alloc(ctx, &p_off, (size_t)(K + 1) * sizeof(int64_t)));
    s.d_off = (int64_t*)p_off;
    LTR_CUDA(ctx, cudaMemcpyAsync(s.d_off, off.data(), (size_t)(K + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `off` may be a temporary
    p_pts = nullptr; p_off = nullptr;
    ctx->scansets[slot] = s;
    *out = ScanSetOwner(ctx, slot);
    return LTR_OK;
}
int scanset_get(ltr_ctx* ctx, ltr_scanset h, DevScanSet** s) {
    if (h < 0 || h >= (int)ctx->scansets.size() || !ctx->scansets[h].used) return fail(ctx, LTR_ERR_INVALID, "invalid scanset handle %d", h);
    *s = &ctx->scansets[h];
    return LTR_OK;
}
int poses_get(ltr_ctx* ctx, ltr_poses h, DevPoses** p) {
    if (h < 0 || h >= (int)ctx->poses.size() || !ctx->poses[h].used) return fail(ctx, LTR_ERR_INVALID, "invalid poses handle %d", h);
    *p = &ctx->poses[h];
    return LTR_OK;
}

// AoS (x,y,z,i) <-> SoA
__global__ void aos_to_soa_kernel(const float4* __restrict__ in, float* __restrict__ x, float* __restrict__ y, float* __restrict__ z,
                                  float* __restrict__ w, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = in[i];
    x[i] = p.x; y[i] = p.y; z[i] = p.z; w[i] = p.w;
}
__global__ void soa_to_aos_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ z,
                                  const float* __restrict__ w, float4* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = make_float4(x[i], y[i], z[i], w[i]);
}

static int upload_points(ltr_ctx* ctx, const float* xyzi, DevCloud& c) {
    if (c.n == 0) return LTR_OK;
    void* stage = nullptr;
    ScratchGuard g_stage(ctx, &stage);
    LTR_TRY(dev_alloc(ctx, &stage, (size_t)c.n * 16));
    LTR_CUDA(ctx, cudaMemcpyAsync(stage, xyzi, (size_t)c.n * 16, cudaMemcpyHostToDevice, ctx->stream));
    const int T = 256;
    aos_to_soa_kernel<<<(unsigned)((c.n + T - 1) / T), T, 0, ctx->stream>>>((const float4*)stage, c.x(), c.y(), c.z(), c.i(), c.n);
    LTR_LAUNCH_CHECK(ctx);
    g_stage.release();
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // caller's host buffer is only read during the call
    return LTR_OK;
}
static int download_points(ltr_ctx* ctx, const DevCloud& c, float* xyzi) {
    if (c.n == 0) return LTR_OK;
    void* stage = nullptr;
    ScratchGuard g_stage(ctx, &stage);
    LTR_TRY(dev_alloc(ctx, &stage, (size_t)c.n * 16));
    const int T = 256;
    soa_to_aos_kernel<<<(unsigned)((c.n + T - 1) / T), T, 0, ctx->stream>>>(c.x(), c.y(), c.z(), c.i(), (float4*)stage, c.n);
    LTR_LAUNCH_CHECK(ctx);
    LTR_CUDA(ctx, cudaMemcpyAsync(xyzi, stage, (size_t)c.n * 16, cudaMemcpyDeviceToHost, ctx->stream));
    g_stage.release();
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}

// KfFast of one keyframe: M = base2lidar * inv_pose (3x4, double); q = A (p - c) = A (p - c_hi) - A c_lo, c = -A^-1 t, c_hi = fl32(c)
static void make_kf_fast(const double* inv_pose /*12*/, const double* b2l /*16*/, bool ext_identity, float* out /*16*/) {
    double M[12];
    if (ext_identity) { for (int i = 0; i < 12; ++i) M[i] = inv_pose[i]; }
    else {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 4; ++c) {
                double v = 0.0;
                for (int j = 0; j < 3; ++j) v += b2l[r * 4 + j] * inv_pose[j * 4 + c];
                if (c == 3) v += b2l[r * 4 + 3];
                M[r * 4 + c] = v;
            }
    }
    const double a = M[0], b = M[1], c = M[2], d = M[4], e = M[5], f = M[6], g = M[8], h = M[9], i = M[10];
    const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
    bool ok = std::isfinite(det) && std::fabs(det) > 1e-6 && std::fabs(det) < 1e6;
    // The error budget of the fast path (project_fast.cuh) and the bounding-sphere / cone bound of the tile culling (project_cull.cuh)
    // assume a RIGID transform: rows of unit length, mutually orthogonal.  A scaled or sheared inverse pose / extrinsic keeps the
    // reference arithmetic only (ok = 0 -> every pair of this keyframe takes the exact path).
    for (int r1 = 0; r1 < 3 && ok; ++r1)
        for (int r2 = r1; r2 < 3; ++r2) {
            const double dot = M[r1 * 4 + 0] * M[r2 * 4 + 0] + M[r1 * 4 + 1] * M[r2 * 4 + 1] + M[r1 * 4 + 2] * M[r2 * 4 + 2];
            if (!(std::fabs(dot - (r1 == r2 ? 1.0 : 0.0)) < 1e-5)) ok = false;
        }
    double inv[9] = {(e * i - f * h), (c * h - b * i), (b * f - c * e), (f * g - d * i), (a * i - c * g), (c * d - a * f), (d * h - e * g), (b * g - a * h), (a * e - b * d)};
    double cc[3] = {0, 0, 0};
    if (ok) for (int r = 0; r < 3; ++r) cc[r] = -(inv[r * 3 + 0] * M[3] + inv[r * 3 + 1] * M[7] + inv[r * 3 + 2] * M[11]) / det;
    for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) { out[r * 3 + k] = (float)M[r * 4 + k]; if (!std::isfinite(out[r * 3 + k])) ok = false; }
    double clo[3];
    for (int r = 0; r < 3; ++r) {
        const float hi = (float)cc[r];
        out[9 + r] = hi;                       // c_hi
        clo[r] = cc[r] - (double)hi;
        if (!std::isfinite(hi)) ok = false;
    }
    for (int r = 0; r < 3; ++r) out[12 + r] = (float)(M[r * 4 + 0] * clo[0] + M[r * 4 + 1] * clo[1] + M[r * 4 + 2] * clo[2]);  // t_lo = A c_lo
    out[15] = ok ? 1.0f : 0.0f;
}

static bool is_identity(const double* m) {
    for (int i = 0; i < 16; ++i) if (m[i] != ((i % 5 == 0) ? 1.0 : 0.0)) return false;
    return true;
}

}  // namespace ltr

using namespace ltr;

extern "C" {

void ltr_config_default(ltr_config* cfg) {
    std::memset(cfg, 0, sizeof(*cfg));
    cfg->device = 0;
    cfg->vfov_deg = 50.0f;
    cfg->hfov_deg = 360.0f;
    for (int i = 0; i < 16; ++i) cfg->lidar2base[i] = cfg->base2lidar[i] = (i % 5 == 0) ? 1.0 : 0.0;
    cfg->transform_order = 0;
    cfg->keyframe_batch = 0;
    cfg->fast_path = 2;
}

int ltr_create(ltr_ctx** out, const ltr_config* cfg) {
    if (!out || !cfg) return fail(nullptr, LTR_ERR_INVALID, "null argument");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return fail(nullptr, LTR_ERR_CUDA, "no CUDA device: %s", cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, LTR_ERR_INVALID, "device %d out of range (%d devices)", cfg->device, ndev);
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, cfg->device);
    if (e != cudaSuccess) return fail(nullptr, LTR_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0) return fail(nullptr, LTR_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
    if (!(cfg->vfov_deg > 0) || !(cfg->hfov_deg > 0)) return fail(nullptr, LTR_ERR_INVALID, "fov must be positive");
    if (cfg->transform_order != 0 && cfg->transform_order != 1) return fail(nullptr, LTR_ERR_INVALID, "transform_order must be 0 or 1");
    e = cudaSetDevice(cfg->device);
    if (e != cudaSuccess) return fail(nullptr, LTR_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
    ltr_ctx* ctx = new ltr_ctx();
    ctx->cfg = *cfg;
    if (ctx->cfg.keyframe_batch <= 0) ctx->cfg.keyframe_batch = 32;
    ctx->device = cfg->device;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->cache_limit_bytes = (size_t)((double)prop.totalGlobalMem * 0.45);   // idle blocks kept for reuse: at most 45 % of the device memory
    ctx->ext_identity = is_identity(cfg->lidar2base) && is_identity(cfg->base2lidar);
    { const char* t = getenv("LTR_TRACE"); ctx->trace = t && t[0] == '1'; }
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&ctx->ev0) != cudaSuccess || cudaEventCreate(&ctx->ev1) != cudaSuccess) {
        delete ctx;
        return fail(nullptr, LTR_ERR_CUDA, "stream/event creation failed");
    }
    cudaEventCreate(&ctx->ev_timer0);
    cudaEventCreate(&ctx->ev_timer1);
    ctx->ev_pool.resize(512);
    for (auto& e2 : ctx->ev_pool) cudaEventCreate(&e2);
    double ext[24];
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 4; ++c) { ext[r * 4 + c] = cfg->base2lidar[r * 4 + c]; ext[12 + r * 4 + c] = cfg->lidar2base[r * 4 + c]; }
    void* p;
    if (dev_alloc(ctx, &p, sizeof(ext)) != LTR_OK) { g_create_err = ctx->err; delete ctx; return LTR_ERR_CUDA; }
    ctx->d_ext = (double*)p;
    cudaMemcpyAsync(ctx->d_ext, ext, sizeof(ext), cudaMemcpyHostToDevice, ctx->stream);
    if (dev_alloc(ctx, &p, 8 * sizeof(unsigned long long)) != LTR_OK) { g_create_err = ctx->err; delete ctx; return LTR_ERR_CUDA; }
    ctx->d_counters = (unsigned long long*)p;
    cudaMemsetAsync(ctx->d_counters, 0, 8 * sizeof(unsigned long long), ctx->stream);
    if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) { delete ctx; return fail(nullptr, LTR_ERR_CUDA, "context initialisation failed"); }
    *out = ctx;
    return LTR_OK;
}

void ltr_destroy(ltr_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->trace) ltr_trace_dump(ctx, 1);
    for (size_t i = 0; i < ctx->nccl.size(); ++i) if (ctx->nccl[i].used) ltr_nccl_destroy(ctx, (int32_t)i);
    scan_images_release(ctx, 0, true);
    for (auto& c : ctx->clouds) if (c.used) cloud_release(ctx, &c);
    for (auto& s : ctx->scansets) if (s.used) { cloud_release(ctx, &s.pts); dev_free(ctx, s.d_off); }
    for (auto& p : ctx->poses) if (p.used) { dev_free(ctx, p.d); dev_free(ctx, p.d_fast); }
    dev_free(ctx, ctx->d_ext);
    dev_free(ctx, ctx->d_counters);
    cudaStreamSynchronize(ctx->stream);
    for (auto& kv : ctx->free_blocks) cudaFree(kv.second);
    for (auto& kv : ctx->live_blocks) cudaFree(kv.first);
    for (auto& e2 : ctx->ev_pool) cudaEventDestroy(e2);
    cudaEventDestroy(ctx->ev_timer0);
    cudaEventDestroy(ctx->ev_timer1);
    cudaEventDestroy(ctx->ev0);
    cudaEventDestroy(ctx->ev1);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* ltr_last_error(const ltr_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int ltr_synchronize(ltr_ctx* ctx) {
    ApiTrace tr__(ctx, "ltr_synchronize");
    if (!ctx) return LTR_ERR_INVALID;
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}

// page-locked host staging memory (full-rate, truly asynchronous H2D / D2H); not tied to a context
int ltr_pinned_alloc(size_t bytes, void** out) {
    if (!out) return LTR_ERR_INVALID;
    *out = nullptr;
    if (bytes == 0) return LTR_OK;
    return cudaMallocHost(out, bytes) == cudaSuccess ? LTR_OK : LTR_ERR_NOMEM;
}
void ltr_pinned_free(void* p) { if (p) cudaFreeHost(p); }

int64_t ltr_kernel_launches(const ltr_ctx* ctx) { return ctx ? ctx->launches : 0; }
void* ltr_stream_handle(ltr_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int64_t ltr_voxel_shortcuts(const ltr_ctx* ctx) { return ctx ? ctx->vox_shortcuts : 0; }
int ltr_memory_stats(const ltr_ctx* ctx, int64_t* stats3) {
    if (!ctx || !stats3) return LTR_ERR_INVALID;
    stats3[0] = (int64_t)ctx->live_bytes; stats3[1] = (int64_t)ctx->cached_bytes; stats3[2] = (int64_t)ctx->peak_live_bytes;
    return LTR_OK;
}

int ltr_cloud_upload(ltr_ctx* ctx, const float* xyzi, int64_t n, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_cloud_upload");
    if (!ctx || !out || (n > 0 && !xyzi)) return fail(ctx, LTR_ERR_INVALID, "null argument");
    CloudOwner o;
    LTR_TRY(cloud_new(ctx, n, &o));
    LTR_TRY(upload_points(ctx, xyzi, ctx->clouds[o.get()]));
    *out = o.release();
    return LTR_OK;
}
int ltr_cloud_alloc(ltr_ctx* ctx, int64_t n, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_cloud_alloc");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    CloudOwner o;
    LTR_TRY(cloud_new(ctx, n, &o));
    *out = o.release();
    return LTR_OK;
}
int ltr_cloud_size(ltr_ctx* ctx, ltr_cloud c, int64_t* n) {
    DevCloud* dc;
    LTR_TRY(cloud_get(ctx, c, &dc));
    *n = dc->n;
    return LTR_OK;
}
int ltr_cloud_download(ltr_ctx* ctx, ltr_cloud c, float* xyzi, int64_t capacity, int64_t* n) {
    ApiTrace tr__(ctx, "ltr_cloud_download");
    DevCloud* dc;
    LTR_TRY(cloud_get(ctx, c, &dc));
    if (n) *n = dc->n;
    if (capacity < dc->n) return fail(ctx, LTR_ERR_INVALID, "download buffer too small (%lld < %lld)", (long long)capacity, (long long)dc->n);
    return download_points(ctx, *dc, xyzi);
}
int ltr_cloud_free(ltr_ctx* ctx, ltr_cloud c) {
    ApiTrace tr__(ctx, "ltr_cloud_free");
    DevCloud* dc;
    LTR_TRY(cloud_get(ctx, c, &dc));
    cloud_release(ctx, dc);
    return LTR_OK;
}
int ltr_cloud_copy(ltr_ctx* ctx, ltr_cloud src, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_cloud_copy");
    DevCloud* s;
    LTR_TRY(cloud_get(ctx, src, &s));
    const DevCloud sc = *s;
    CloudOwner o;
    LTR_TRY(cloud_new(ctx, sc.n, &o));
    DevCloud& d = ctx->clouds[o.get()];
    if (sc.n > 0) {
        LTR_CUDA(ctx, cudaMemcpy2DAsync(d.base, (size_t)d.cap * 4, sc.base, (size_t)sc.cap * 4, (size_t)sc.n * 4, 4, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    *out = o.release();
    return LTR_OK;
}
int ltr_cloud_slice(ltr_ctx* ctx, ltr_cloud src, int64_t begin, int64_t end, ltr_cloud* out) {
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevCloud* s;
    LTR_TRY(cloud_get(ctx, src, &s));
    if (begin < 0 || end < begin || end > s->n) return fail(ctx, LTR_ERR_INVALID, "slice [%lld, %lld) outside [0, %lld)", (long long)begin, (long long)end, (long long)s->n);
    DevCloud v = *s;
    v.base = s->base + begin; v.n = end - begin; v.flags = nullptr; v.borrowed = true;   // same component stride (cap)
    int slot = -1;
    for (size_t i = 0; i < ctx->clouds.size(); ++i) if (!ctx->clouds[i].used) { slot = (int)i; break; }
    if (slot < 0) { ctx->clouds.push_back(DevCloud()); slot = (int)ctx->clouds.size() - 1; }
    ctx->clouds[slot] = v;
    *out = slot;
    return LTR_OK;
}
int ltr_cloud_concat(ltr_ctx* ctx, ltr_cloud a, ltr_cloud b, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_cloud_concat");
    DevCloud *pa, *pb;
    LTR_TRY(cloud_get(ctx, a, &pa));
    LTR_TRY(cloud_get(ctx, b, &pb));
    const DevCloud ca = *pa, cb = *pb;
    CloudOwner o;
    LTR_TRY(cloud_new(ctx, ca.n + cb.n, &o));
    DevCloud& d = ctx->clouds[o.get()];
    if (ca.n > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(d.base, (size_t)d.cap * 4, ca.base, (size_t)ca.cap * 4, (size_t)ca.n * 4, 4, cudaMemcpyDeviceToDevice, ctx->stream));
    if (cb.n > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(d.base + ca.n, (size_t)d.cap * 4, cb.base, (size_t)cb.cap * 4, (size_t)cb.n * 4, 4, cudaMemcpyDeviceToDevice, ctx->stream));
    *out = o.release();
    return LTR_OK;
}
int ltr_cloud_device_ptrs(ltr_ctx* ctx, ltr_cloud c, float** x, float** y, float** z, float** i, int64_t* n) {
    DevCloud* dc;
    LTR_TRY(cloud_get(ctx, c, &dc));
    if (x) *x = dc->x();
    if (y) *y = dc->y();
    if (z) *z = dc->z();
    if (i) *i = dc->i();
    if (n) *n = dc->n;
    return LTR_OK;
}

int ltr_scanset_upload(ltr_ctx* ctx, const float* xyzi, const int64_t* offsets, int32_t K, ltr_scanset* out) {
    ApiTrace tr__(ctx, "ltr_scanset_upload");
    if (!ctx || !out || !offsets || K < 0) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    std::vector<int64_t> off(offsets, offsets + K + 1);
    if (off[K] > 0 && !xyzi) return fail(ctx, LTR_ERR_INVALID, "null points");
    ScanSetOwner o;
    LTR_TRY(scanset_new(ctx, off, &o));
    LTR_TRY(upload_points(ctx, xyzi, ctx->scansets[o.get()].pts));
    *out = o.release();
    return LTR_OK;
}
int ltr_scanset_info(ltr_ctx* ctx, ltr_scanset s, int32_t* K, int64_t* total) {
    DevScanSet* ss;
    LTR_TRY(scanset_get(ctx, s, &ss));
    if (K) *K = ss->K;
    if (total) *total = ss->pts.n;
    return LTR_OK;
}
int ltr_scanset_download(ltr_ctx* ctx, ltr_scanset s, float* xyzi, int64_t capacity, int64_t* offsets) {
    ApiTrace tr__(ctx, "ltr_scanset_download");
    DevScanSet* ss;
    LTR_TRY(scanset_get(ctx, s, &ss));
    if (offsets) std::memcpy(offsets, ss->h_off.data(), (size_t)(ss->K + 1) * sizeof(int64_t));
    if (!xyzi) return LTR_OK;
    if (capacity < ss->pts.n) return fail(ctx, LTR_ERR_INVALID, "download buffer too small");
    return download_points(ctx, ss->pts, xyzi);
}
int ltr_scanset_free(ltr_ctx* ctx, ltr_scanset s) {
    ApiTrace tr__(ctx, "ltr_scanset_free");
    DevScanSet* ss;
    LTR_TRY(scanset_get(ctx, s, &ss));
    scan_images_release(ctx, ss->serial, false);
    cloud_release(ctx, &ss->pts);
    dev_free(ctx, ss->d_off);
    *ss = DevScanSet();
    return LTR_OK;
}
int ltr_scanset_flatten(ltr_ctx* ctx, ltr_scanset s, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_scanset_flatten");
    DevScanSet* ss;
    LTR_TRY(scanset_get(ctx, s, &ss));
    const DevCloud sc = ss->pts;
    CloudOwner o;
    LTR_TRY(cloud_new(ctx, sc.n, &o));
    DevCloud& d = ctx->clouds[o.get()];
    if (sc.n > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(d.base, (size_t)d.cap * 4, sc.base, (size_t)sc.cap * 4, (size_t)sc.n * 4, 4, cudaMemcpyDeviceToDevice, ctx->stream));
    *out = o.release();
    return LTR_OK;
}
int ltr_scanset_concat_per_keyframe(ltr_ctx* ctx, ltr_scanset a, ltr_scanset b, ltr_scanset* out) {
    ApiTrace tr__(ctx, "ltr_scanset_concat_per_keyframe");
    DevScanSet *pa, *pb;
    LTR_TRY(scanset_get(ctx, a, &pa));
    LTR_TRY(scanset_get(ctx, b, &pb));
    if (pa->K != pb->K) return fail(ctx, LTR_ERR_INVALID, "scansets have different keyframe counts (%d vs %d)", pa->K, pb->K);
    const int K = pa->K;
    std::vector<int64_t> off((size_t)K + 1, 0);
    for (int k = 0; k < K; ++k) off[k + 1] = off[k] + (pa->h_off[k + 1] - pa->h_off[k]) + (pb->h_off[k + 1] - pb->h_off[k]);
    const DevCloud ca = pa->pts, cb = pb->pts;
    const std::vector<int64_t> oa = pa->h_off, ob = pb->h_off;
    ScanSetOwner o;
    LTR_TRY(scanset_new(ctx, off, &o));
    DevCloud& d = ctx->scansets[o.get()].pts;
    for (int k = 0; k < K; ++k) {
        const int64_t na = oa[k + 1] - oa[k], nb = ob[k + 1] - ob[k];
        if (na > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(d.base + off[k], (size_t)d.cap * 4, ca.base + oa[k], (size_t)ca.cap * 4, (size_t)na * 4, 4, cudaMemcpyDeviceToDevice, ctx->stream));
        if (nb > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(d.base + off[k] + na, (size_t)d.cap * 4, cb.base + ob[k], (size_t)cb.cap * 4, (size_t)nb * 4, 4, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    *out = o.release();
    return LTR_OK;
}

int ltr_poses_upload(ltr_ctx* ctx, const double* poses, const double* inv_poses, int32_t K, ltr_poses* out) {
    ApiTrace tr__(ctx, "ltr_poses_upload");
    if (!ctx || !out || K < 0 || (K > 0 && (!poses || !inv_poses))) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    int slot = -1;
    for (size_t i = 0; i < ctx->poses.size(); ++i) if (!ctx->poses[i].used) { slot = (int)i; break; }
    if (slot < 0) { ctx->poses.push_back(DevPoses()); slot = (int)ctx->poses.size() - 1; }
    DevPoses p;
    p.K = K; p.used = true; p.serial = ++ctx->next_serial;
    p.h.resize((size_t)K * 24);
    for (int k = 0; k < K; ++k) {
        std::memcpy(&p.h[(size_t)k * 24], inv_poses + (size_t)k * 16, 12 * sizeof(double));
        std::memcpy(&p.h[(size_t)k * 24 + 12], poses + (size_t)k * 16, 12 * sizeof(double));
    }
    void *p_d = nullptr, *p_fast = nullptr;
    ScratchGuard g_d(ctx, &p_d), g_fast(ctx, &p_fast);   // disarmed once the handle owns both blocks
    LTR_TRY(dev_alloc(ctx, &p_d, (size_t)K * 24 * sizeof(double)));
    p.d = (double*)p_d;
    if (K > 0) LTR_CUDA(ctx, cudaMemcpyAsync(p.d, p.h.data(), (size_t)K * 24 * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    p.h_fast.resize((size_t)K * 16);
    for (int k = 0; k < K; ++k) make_kf_fast(&p.h[(size_t)k * 24], ctx->cfg.base2lidar, ctx->ext_identity, &p.h_fast[(size_t)k * 16]);
    LTR_TRY(dev_alloc(ctx, &p_fast, (size_t)K * 16 * sizeof(float)));
    p.d_fast = (float*)p_fast;
    if (K > 0) LTR_CUDA(ctx, cudaMemcpyAsync(p.d_fast, p.h_fast.data(), (size_t)K * 16 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    p_d = p_fast = nullptr;
    ctx->poses[slot] = p;
    *out = slot;
    return LTR_OK;
}
int ltr_poses_free(ltr_ctx* ctx, ltr_poses h) {
    ApiTrace tr__(ctx, "ltr_poses_free");
    DevPoses* p;
    LTR_TRY(poses_get(ctx, h, &p));
    scan_images_release(ctx, p->serial, false);
    dev_free(ctx, p->d);
    dev_free(ctx, p->d_fast);
    *p = DevPoses();
    return LTR_OK;
}

void ltr_reset_rimg_size(float vfov, float hfov, float alpha, int32_t* rows, int32_t* cols) {
    // resetRimgSize (utility.cpp:222-236): int = std::round(float * float)
    *rows = (int32_t)roundf(vfov * alpha);
    *cols = (int32_t)roundf(hfov * alpha);
}

int ltr_profile_get(ltr_ctx* ctx, double* out8) {
    if (!ctx || !out8) return LTR_ERR_INVALID;
    for (int i = 0; i < 8; ++i) out8[i] = ctx->prof[i];
    return LTR_OK;
}
int ltr_profile_reset(ltr_ctx* ctx) {
    if (!ctx) return LTR_ERR_INVALID;
    for (int i = 0; i < 8; ++i) ctx->prof[i] = 0.0;
    return LTR_OK;
}

int ltr_trace_dump(ltr_ctx* ctx, int reset) {
    if (!ctx) return LTR_ERR_INVALID;
    double tot = 0;
    for (auto& kv : ctx->trace_acc) tot += kv.second.first;
    fprintf(stderr, "[ltr alloc] live %.2f GB (peak %.2f GB), cached %.2f GB in %zu blocks, cudaMalloc calls %ld, cache hits %ld, purges %ld\n", ctx->live_bytes / 1e9,
            ctx->peak_live_bytes / 1e9, ctx->cached_bytes / 1e9, ctx->free_blocks.size(), ctx->n_cuda_malloc, ctx->n_cache_hits, ctx->n_purges);
    fprintf(stderr, "[ltr trace] total %.2f ms in %zu entry points\n", tot * 1e3, ctx->trace_acc.size());
    for (auto& kv : ctx->trace_acc) fprintf(stderr, "[ltr trace] %-36s calls %6ld  %10.3f ms\n", kv.first.c_str(), kv.second.second, kv.second.first * 1e3);
    if (reset) ctx->trace_acc.clear();
    return LTR_OK;
}

int ltr_timer_start(ltr_ctx* ctx) {
    ApiTrace tr__(ctx, "ltr_timer_start");
    if (!ctx) return LTR_ERR_INVALID;
    LTR_CUDA(ctx, cudaEventRecord(ctx->ev_timer0, ctx->stream));
    return LTR_OK;
}
int ltr_timer_stop(ltr_ctx* ctx, double* ms) {
    ApiTrace tr__(ctx, "ltr_timer_stop");
    if (!ctx || !ms) return LTR_ERR_INVALID;
    LTR_CUDA(ctx, cudaEventRecord(ctx->ev_timer1, ctx->stream));
    LTR_CUDA(ctx, cudaEventSynchronize(ctx->ev_timer1));
    float f = 0.0f;
    LTR_CUDA(ctx, cudaEventElapsedTime(&f, ctx->ev_timer0, ctx->ev_timer1));
    *ms = (double)f;
    return LTR_OK;
}

int ltr_last_pass_stats(ltr_ctx* ctx, double* s) {
    ApiTrace tr__(ctx, "ltr_last_pass_stats");
    if (!ctx || !s) return LTR_ERR_INVALID;
    if (ctx->stats_counters_pending) {
        unsigned long long c[4] = {0, 0, 0, 0};
        LTR_CUDA(ctx, cudaMemcpyAsync(c, ctx->d_counters, sizeof(c), cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        ctx->stats[2] = (double)c[0] + (double)c[2];  // pairs that needed exact arithmetic (range-only + full)
        ctx->stats[1] = ctx->stats[0] - ctx->stats[2];
        ctx->stats[3] = (double)c[1];
        ctx->stats[5] = (double)c[2];                 // pairs through the FULL exact path
        ctx->stats[6] = (double)c[3];                 // pairs skipped by tile culling
        ctx->stats_counters_pending = false;
    }
    for (int i = 0; i < 7; ++i) s[i] = ctx->stats[i];
    return LTR_OK;
}

}  // extern "C"
