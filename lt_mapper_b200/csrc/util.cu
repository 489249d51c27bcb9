// libltr_b200.so -- order-preserving compaction, reductions, voxel centroid, merge and pre-clean kernels.
#include "ltr_internal.cuh"
#include "ref_math.cuh"
#include "device_util.cuh"
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <algorithm>
#include <deque>

namespace ltr {

constexpr int kPartThreads = 256;
constexpr int kPartRounds = 8;
constexpr int kPartTile = kPartThreads * kPartRounds;

__global__ void __launch_bounds__(kPartThreads) part_count_kernel(const uint8_t* __restrict__ flags, int64_t n, uint32_t* __restrict__ block_cnt) {
    __shared__ int s_warp[33];
    const int64_t base = (int64_t)blockIdx.x * kPartTile;
    int cnt = 0;
#pragma unroll
    for (int r = 0; r < kPartRounds; ++r) {
        const int64_t i = base + (int64_t)r * kPartThreads + threadIdx.x;
        cnt += (i < n && flags[i]) ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kPartThreads / 32; ++w) t += s_warp[w];
        block_cnt[blockIdx.x] = (uint32_t)t;
    }
}

// single-block exclusive scan of up to 2^31 total over nb block counts; writes total to out[nb]
__global__ void __launch_bounds__(1024) scan_blocks_kernel(const uint32_t* in, uint32_t* out, int nb)   /* in may alias out */ {
    __shared__ int s_warp[33];
    __shared__ uint32_t s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int b0 = 0; b0 < nb; b0 += 1024) {
        const int i = b0 + threadIdx.x;
        const uint32_t v = i < nb ? in[i] : 0u;
        // inclusive warp scan
        uint32_t incl = v;
        const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += t; }
        if (lane == 31) s_warp[warp] = (int)incl;
        __syncthreads();
        if (warp == 0) {
            int w = s_warp[lane];
            int wi = w;
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if ((int)lane >= o) wi += t; }
            s_warp[lane] = wi - w;
            if (lane == 31) s_warp[32] = wi;
        }
        __syncthreads();
        const uint32_t excl = s_carry + (uint32_t)s_warp[warp] + incl - v;
        if (i < nb) out[i] = excl;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += (uint32_t)s_warp[32];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[nb] = s_carry;
}

__global__ void __launch_bounds__(kPartThreads) part_scatter_kernel(PtrView in, const uint8_t* __restrict__ flags,
                                                                    const uint32_t* __restrict__ block_off, DevCloud out0, DevCloud out1) {
    __shared__ int s_warp[33];
    const int64_t base = (int64_t)blockIdx.x * kPartTile;
    int64_t dyn_before = block_off[blockIdx.x];
#pragma unroll 1
    for (int r = 0; r < kPartRounds; ++r) {
        const int64_t i = base + (int64_t)r * kPartThreads + threadIdx.x;
        const bool valid = i < in.n;
        const bool f = valid && flags[i];
        int total;
        const int rk = block_rank(f, &total, s_warp);
        if (valid) {
            const float x = in.x[i], y = in.y[i], z = in.z[i], w = in.i[i];
            if (f) {
                const int64_t o = dyn_before + rk;
                out1.x()[o] = x; out1.y()[o] = y; out1.z()[o] = z; out1.i()[o] = w;
            } else {
                const int64_t o = i - (dyn_before + rk);
                out0.x()[o] = x; out0.y()[o] = y; out0.z()[o] = z; out0.i()[o] = w;
            }
        }
        dyn_before += total;
    }
}

int stable_partition_by_flag(ltr_ctx* ctx, const DevCloud& in, const uint8_t* flags, int64_t* n_flagged, DevCloud* out0, DevCloud* out1) {
    const int64_t n = in.n;
    if (n == 0) { *n_flagged = 0; out0->n = 0; out1->n = 0; return LTR_OK; }
    const int nb = (int)((n + kPartTile - 1) / kPartTile);
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, (size_t)(2 * nb + 2) * sizeof(uint32_t)));
    uint32_t* cnt = (uint32_t*)p;
    uint32_t* off = cnt + nb;
    part_count_kernel<<<nb, kPartThreads, 0, ctx->stream>>>(flags, n, cnt);
    LTR_LAUNCH_CHECK(ctx);
    scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(cnt, off, nb);
    LTR_LAUNCH_CHECK(ctx);
    part_scatter_kernel<<<nb, kPartThreads, 0, ctx->stream>>>(view(in), flags, off, *out0, *out1);
    LTR_LAUNCH_CHECK(ctx);
    uint32_t total = 0;
    LTR_CUDA(ctx, cudaMemcpyAsync(&total, off + nb, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    g_p.release();
    *n_flagged = total;
    out1->n = total;
    out0->n = n - total;
    return LTR_OK;
}

int count_flags(ltr_ctx* ctx, const uint8_t* flags, int64_t n, int64_t* count) {
    if (n == 0) { *count = 0; return LTR_OK; }
    const int nb = (int)((n + kPartTile - 1) / kPartTile);
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, (size_t)(2 * nb + 2) * sizeof(uint32_t)));
    uint32_t* cnt = (uint32_t*)p;
    part_count_kernel<<<nb, kPartThreads, 0, ctx->stream>>>(flags, n, cnt);
    LTR_LAUNCH_CHECK(ctx);
    scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(cnt, cnt + nb, nb);
    LTR_LAUNCH_CHECK(ctx);
    uint32_t total = 0;
    LTR_CUDA(ctx, cudaMemcpyAsync(&total, cnt + 2 * nb, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    g_p.release();
    *count = total;
    return LTR_OK;
}

// ------------------------------------------------------------------------------------------------
// Device-wide exclusive prefix sum of u32 (reduce - scan - apply; in and out may alias).  Used for the kNN grid's cell starts,
// the voxel ranks and the digit offsets of the radix sort below.
// ------------------------------------------------------------------------------------------------
constexpr int kScanThreads = 1024;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(const uint32_t* __restrict__ in, int64_t n, uint32_t* __restrict__ part) {
    __shared__ uint32_t s_warp[32];
    const int64_t base = (int64_t)blockIdx.x * kScanTile;
    uint32_t sum = 0;
#pragma unroll
    for (int r = 0; r < kScanItems; ++r) {
        const int64_t i = base + (int64_t)r * kScanThreads + threadIdx.x;
        if (i < n) sum += in[i];
    }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x < 32) {
        sum = s_warp[threadIdx.x];
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_down_sync(0xffffffffu, sum, o);
        if (threadIdx.x == 0) part[blockIdx.x] = sum;
    }
}

// each thread owns kScanItems CONSECUTIVE elements (blocked arrangement), so the scan order is the element order
__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(const uint32_t* in, uint32_t* out, int64_t n,   /* in may alias out */
                                                                  const uint32_t* __restrict__ part_excl) {
    __shared__ uint32_t s_warp[33];
    const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    uint32_t v[kScanItems];
    uint32_t sum = 0;
#pragma unroll
    for (int r = 0; r < kScanItems; ++r) { const int64_t i = base + r; v[r] = i < n ? in[i] : 0u; sum += v[r]; }
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = sum;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += t; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = s_warp[lane];
        uint32_t wi = w;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, wi, o); if ((int)lane >= o) wi += t; }
        s_warp[lane] = wi - w;
    }
    __syncthreads();
    uint32_t run = part_excl[blockIdx.x] + s_warp[warp] + incl - sum;
#pragma unroll
    for (int r = 0; r < kScanItems; ++r) { const int64_t i = base + r; if (i < n) out[i] = run; run += v[r]; }
}

int exclusive_scan_u32(ltr_ctx* ctx, const uint32_t* in, uint32_t* out, int64_t n) {
    if (n <= 0) return LTR_OK;
    const int nb = (int)((n + kScanTile - 1) / kScanTile);
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, (size_t)(2 * nb + 2) * sizeof(uint32_t)));
    uint32_t* part = (uint32_t*)p;
    uint32_t* part_excl = part + nb;
    scan_reduce_kernel<<<nb, kScanThreads, 0, ctx->stream>>>(in, n, part);
    LTR_LAUNCH_CHECK(ctx);
    scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(part, part_excl, nb);
    LTR_LAUNCH_CHECK(ctx);
    scan_apply_kernel<<<nb, kScanThreads, 0, ctx->stream>>>(in, out, n, part_excl);
    LTR_LAUNCH_CHECK(ctx);
    g_p.release();
    return LTR_OK;
}

// ------------------------------------------------------------------------------------------------
// Stable LSD radix sort of (u64 key, u32 value) pairs on the key bits [0, key_bits), 8 bits per pass (the voxeliser's Morton sort).
// Per pass: per-tile digit histogram -> exclusive scan of the digit-major [256][tiles] matrix -> stable scatter.  Stability inside a
// tile: every warp owns a CONTIGUOUS run of the tile and walks it 32 elements at a time; __match_any_sync gives each element its rank
// among the equal digits of its row, per-warp running counters give the rank among the earlier rows, and a prefix over the warps of
// the tile gives the rank among the earlier warps.  Equal keys therefore keep their input order, which is what makes the voxel
// sums run in insertion order (PCL's leaf containers accumulate in insertion order).
// ------------------------------------------------------------------------------------------------
constexpr int kRsThreads = 256;
constexpr int kRsItems = 16;
constexpr int kRsTile = kRsThreads * kRsItems;   // 4096 keys per tile, 512 per warp

__global__ void __launch_bounds__(kRsThreads) rs_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift, uint32_t* __restrict__ hist, int ntiles) {
    __shared__ uint32_t s_hist[256];
    s_hist[threadIdx.x] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * kRsTile;
#pragma unroll 4
    for (int r = 0; r < kRsItems; ++r) {
        const int64_t i = base + (int64_t)r * kRsThreads + threadIdx.x;
        if (i < n) atomicAdd(&s_hist[(unsigned)(keys[i] >> shift) & 255u], 1u);
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * ntiles + blockIdx.x] = s_hist[threadIdx.x];
}

// kVals = false: keys only (the voxeliser packs the point index into the low bits of the key whenever both fit 64 bits: 8 instead of
// 12 bytes per element and pass, 32 instead of 48 KB of shared memory per tile)
template <bool kVals>
__global__ void __launch_bounds__(kRsThreads) rs_scatter_kernel(const uint64_t* __restrict__ keys_in, uint64_t* __restrict__ keys_out,
                                                                const uint32_t* __restrict__ vals_in, uint32_t* __restrict__ vals_out, int64_t n, int shift,
                                                                const uint32_t* __restrict__ offs, int ntiles) {
    // dynamic shared memory: the tile's keys and values in their sorted-by-digit order, so that the global writes of a digit bucket
    // are one contiguous, coalesced run instead of 8-byte scatters
    extern __shared__ uint64_t s_keys[];                            // kRsTile keys, then (kVals) kRsTile values
    uint32_t* s_vals = reinterpret_cast<uint32_t*>(s_keys + kRsTile);
    __shared__ uint32_t s_cnt[kRsThreads / 32][256];
    __shared__ uint32_t s_excl[256];     // exclusive prefix of the tile's digit counts (position of the bucket inside the tile)
    __shared__ uint32_t s_gdelta[256];   // global start of the bucket minus its position inside the tile
    __shared__ uint32_t s_wsum[8];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t = threadIdx.x; t < (kRsThreads / 32) * 256; t += kRsThreads) (&s_cnt[0][0])[t] = 0;
    __syncthreads();
    const int64_t tile_base = (int64_t)blockIdx.x * kRsTile;
    const int64_t chunk = tile_base + (int64_t)warp * (32 * kRsItems);
    const int tile_n = (int)min((int64_t)kRsTile, n - tile_base);
    uint64_t key[kRsItems];
    uint32_t rank[kRsItems];
    const unsigned lt = (1u << lane) - 1u;
#pragma unroll
    for (int r = 0; r < kRsItems; ++r) {
        const int64_t i = chunk + r * 32 + lane;
        const bool valid = i < n;
        key[r] = valid ? keys_in[i] : 0ull;
        const unsigned d = (unsigned)(key[r] >> shift) & 255u;
        const unsigned peers = __match_any_sync(0xffffffffu, valid ? d : (256u + lane));   // padding lanes match nobody
        const int leader = __ffs(peers) - 1;
        uint32_t old = 0;
        if ((int)lane == leader && valid) { old = s_cnt[warp][d]; s_cnt[warp][d] = old + __popc(peers); }
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[r] = old + __popc(peers & lt);
        __syncwarp();
    }
    __syncthreads();
    {   // per digit (one per thread): exclusive prefix over the warps, tile total; then an exclusive prefix over the digits
        const int d = threadIdx.x;
        uint32_t sum = 0;
#pragma unroll
        for (int w = 0; w < kRsThreads / 32; ++w) { const uint32_t c = s_cnt[w][d]; s_cnt[w][d] = sum; sum += c; }
        uint32_t incl = sum;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += t; }
        if (lane == 31) s_wsum[warp] = incl;
        __syncthreads();
        uint32_t wbase = 0;
        for (int w = 0; w < (int)warp; ++w) wbase += s_wsum[w];
        const uint32_t excl = wbase + incl - sum;
        s_excl[d] = excl;
        s_gdelta[d] = offs[(size_t)d * ntiles + blockIdx.x] - excl;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kRsItems; ++r) {
        const int64_t i = chunk + r * 32 + lane;
        if (i < n) {
            const unsigned d = (unsigned)(key[r] >> shift) & 255u;
            const uint32_t lp = s_excl[d] + s_cnt[warp][d] + rank[r];
            s_keys[lp] = key[r];
            if (kVals) s_vals[lp] = vals_in[i];
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < tile_n; t += kRsThreads) {
        const uint64_t k = s_keys[t];
        const uint32_t pos = s_gdelta[(unsigned)(k >> shift) & 255u] + (uint32_t)t;
        keys_out[pos] = k;
        if (kVals) vals_out[pos] = s_vals[t];
    }
}

constexpr size_t kRsScatterSmem = (size_t)kRsTile * (sizeof(uint64_t) + sizeof(uint32_t));   // 48 KB: needs the opt-in above 48 KB - 0
constexpr size_t kRsScatterSmemKeys = (size_t)kRsTile * sizeof(uint64_t);                     // 32 KB

// Sorts (keys0, vals0) on the key bits [bit_lo, bit_hi) using (keys1, vals1) as the other half of the ping-pong; *keys_sorted /
// *vals_sorted point at the result.  vals0 == nullptr: keys only.
int radix_sort_pairs(ltr_ctx* ctx, uint64_t* keys0, uint64_t* keys1, uint32_t* vals0, uint32_t* vals1, int64_t n, int bit_lo, int bit_hi,
                            uint64_t** keys_sorted, uint32_t** vals_sorted) {
    *keys_sorted = keys0;
    if (vals_sorted) *vals_sorted = vals0;
    if (n <= 1 || bit_hi <= bit_lo) return LTR_OK;
    const bool with_vals = vals0 != nullptr;
    if (with_vals && !ctx->rs_attr_set) {   // 48 KB dynamic + ~10 KB static shared memory: above the default 48 KB limit (per device)
        LTR_CUDA(ctx, cudaFuncSetAttribute(rs_scatter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRsScatterSmem));
        ctx->rs_attr_set = true;
    }
    const int ntiles = (int)((n + kRsTile - 1) / kRsTile);
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, ((size_t)256 * ntiles + 1) * sizeof(uint32_t)));
    uint32_t* hist = (uint32_t*)p;
    uint64_t *kin = keys0, *kout = keys1;
    uint32_t *vin = vals0, *vout = vals1;
    for (int shift = bit_lo; shift < bit_hi; shift += 8) {
        rs_hist_kernel<<<ntiles, kRsThreads, 0, ctx->stream>>>(kin, n, shift, hist, ntiles);
        LTR_LAUNCH_CHECK(ctx);
        if ((int64_t)256 * ntiles <= 1024 * 64) {   // small matrix: one block scans it (also writes the total past the end, hence the + 1 above)
            scan_blocks_kernel<<<1, 1024, 0, ctx->stream>>>(hist, hist, 256 * ntiles);
            LTR_LAUNCH_CHECK(ctx);
        } else LTR_TRY(exclusive_scan_u32(ctx, hist, hist, (int64_t)256 * ntiles));
        if (with_vals) rs_scatter_kernel<true><<<ntiles, kRsThreads, kRsScatterSmem, ctx->stream>>>(kin, kout, vin, vout, n, shift, hist, ntiles);
        else rs_scatter_kernel<false><<<ntiles, kRsThreads, kRsScatterSmemKeys, ctx->stream>>>(kin, kout, nullptr, nullptr, n, shift, hist, ntiles);
        LTR_LAUNCH_CHECK(ctx);
        std::swap(kin, kout); std::swap(vin, vout);
    }
    g_p.release();
    *keys_sorted = kin;
    if (vals_sorted) *vals_sorted = vin;
    return LTR_OK;
}

// ------------------------------------------------------------------------------------------------
// min / max of x, y, z (pcl::getMinMax3D inside OctreePointCloud::defineBoundingBox)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t f2ord(float f) { const uint32_t u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
static inline float ord2f(uint32_t o) {
    const uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
    float f; memcpy(&f, &u, 4); return f;
}

// nonfinite (may be null): incremented by the number of points with a non-finite x, y or z.  fminf / fmaxf skip NaN, so the
// extrema alone do not reveal them (an all-NaN cloud gives min FLT_MAX and max -FLT_MAX).
__global__ void __launch_bounds__(256) minmax_kernel(PtrView c, uint32_t* __restrict__ out /* 6: min xyz, max xyz (ordered encoding) */,
                                                     uint32_t* __restrict__ nonfinite) {
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    uint32_t bad = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < c.n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = c.x[i], y = c.y[i], z = c.z[i];
        mn[0] = fminf(mn[0], x); mn[1] = fminf(mn[1], y); mn[2] = fminf(mn[2], z);
        mx[0] = fmaxf(mx[0], x); mx[1] = fmaxf(mx[1], y); mx[2] = fmaxf(mx[2], z);
        bad += (isfinite(x) && isfinite(y) && isfinite(z)) ? 0u : 1u;
    }
    for (int d = 0; d < 3; ++d)
        for (int o = 16; o > 0; o >>= 1) {
            mn[d] = fminf(mn[d], __shfl_down_sync(0xffffffffu, mn[d], o));
            mx[d] = fmaxf(mx[d], __shfl_down_sync(0xffffffffu, mx[d], o));
        }
    for (int o = 16; o > 0; o >>= 1) bad += __shfl_down_sync(0xffffffffu, bad, o);
    if ((threadIdx.x & 31) == 0) {
        for (int d = 0; d < 3; ++d) { atomicMin(&out[d], f2ord(mn[d])); atomicMax(&out[3 + d], f2ord(mx[d])); }
        if (nonfinite && bad) atomicAdd(nonfinite, bad);
    }
}

static int minmax_view(ltr_ctx* ctx, const PtrView& v, float mn[3], float mx[3], uint32_t* nonfinite) {
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, 7 * sizeof(uint32_t)));
    uint32_t init[7] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u};
    LTR_CUDA(ctx, cudaMemcpyAsync(p, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    const int blocks = (int)std::min<int64_t>((v.n + 255) / 256, (int64_t)ctx->sm_count * 8);
    minmax_kernel<<<std::max(blocks, 1), 256, 0, ctx->stream>>>(v, (uint32_t*)p, (uint32_t*)p + 6);
    LTR_LAUNCH_CHECK(ctx);
    uint32_t res[7];
    LTR_CUDA(ctx, cudaMemcpyAsync(res, p, sizeof(res), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    g_p.release();
    for (int d = 0; d < 3; ++d) { mn[d] = ord2f(res[d]); mx[d] = ord2f(res[3 + d]); }
    if (nonfinite) *nonfinite = res[6];
    return LTR_OK;
}

int minmax_xyz(ltr_ctx* ctx, const DevCloud& c, float mn[3], float mx[3], uint32_t* nonfinite) { return minmax_view(ctx, view(c), mn, mx, nonfinite); }

int finite_extent(ltr_ctx* ctx, const DevCloud& c, const char* what, float mn[3], float mx[3], const char* where) {
    uint32_t nonfinite = 0;
    LTR_TRY(minmax_xyz(ctx, c, mn, mx, &nonfinite));
    if (nonfinite) return fail(ctx, LTR_ERR_UNSUPPORTED, "non-finite %s coordinates (%u points%s)", what, nonfinite, where);
    return LTR_OK;
}

int check_pose_range(ltr_ctx* ctx, const DevScanSet& scans, const DevPoses& poses, int32_t pose_offset) {
    if (pose_offset < 0 || pose_offset + scans.K > poses.K)
        return fail(ctx, LTR_ERR_INVALID, "pose range [%d,%d) outside [0,%d)", pose_offset, pose_offset + scans.K, poses.K);
    return LTR_OK;
}

__global__ void __launch_bounds__(256) relative_offsets_kernel(const int64_t* __restrict__ off, int kf0, int nkf, int64_t* __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j <= nkf) out[j] = off[kf0 + j] - off[kf0];
}

int relative_offsets(ltr_ctx* ctx, const int64_t* off, int kf0, int nkf, int64_t* out) {
    relative_offsets_kernel<<<(nkf + 1 + 255) / 256, 256, 0, ctx->stream>>>(off, kf0, nkf, out);
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

// ------------------------------------------------------------------------------------------------
// Voxel centroid == pcl::octree::OctreePointCloudVoxelCentroid as used by octreeDownsampling
// (ltremovert/src/utility.cpp:204-219).  PCL semantics (published PCL 1.10 sources, see DESIGN.md):
//   bounding box from min/max (max padded by 512*FLT_EPSILON in f32), grown to a cube of side
//   2^depth*res and centred; key = (unsigned)(((double)p - min) / res); centroid = f32 sums in
//   insertion order / (float)count; output order = octree DFS = ascending Morton code with x as the
//   most significant bit of each level.
// GPU: key -> 3*depth-bit Morton code -> stable LSD radix sort (code, index) -> run heads -> one thread
// per voxel sums its run sequentially in original index order (bit-exact f32 sums).
// ------------------------------------------------------------------------------------------------
struct VoxBox { double min[3]; double res; int depth; };

static VoxBox define_box(const float mn[3], const float mx[3], float leaf) {
    // OctreePointCloud::defineBoundingBox() + getKeyBitSize()
    VoxBox b;
    b.res = (double)leaf;
    const float pad = FLT_EPSILON * 512.0f;
    const float eps = FLT_EPSILON;
    double lo[3], hi[3];
    unsigned mk[3];
    for (int d = 0; d < 3; ++d) {
        const float hf = mx[d] + pad;  // float add
        lo[d] = (double)mn[d];
        hi[d] = (double)hf;
        const double a = std::min(lo[d], hi[d]);
        const double c = std::max(a, hi[d]);
        lo[d] = a; hi[d] = c;
        mk[d] = (unsigned)std::ceil((hi[d] - lo[d] - eps) / b.res);
    }
    const unsigned max_voxels = std::max(std::max(std::max(mk[0], mk[1]), mk[2]), 2u);
    const double lg = std::log((double)max_voxels) / std::log(2.0);
    b.depth = (int)std::max(std::min(32u, (unsigned)std::ceil(lg - eps)), 0u);
    const double side = (double)(1u << b.depth) * b.res;
    for (int d = 0; d < 3; ++d) {
        const double over = (side - (hi[d] - lo[d])) / 2.0;
        if (over > eps) { lo[d] -= over; hi[d] += over; }
        b.min[d] = lo[d];
    }
    return b;
}

__device__ __forceinline__ uint64_t spread3(uint32_t v) {  // 21 bits -> every third bit
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

__device__ __forceinline__ uint64_t vox_code(const PtrView& c, const VoxBox& b, int64_t i, bool* inside) {
    const double fx = __ddiv_rn(__dsub_rn((double)c.x[i], b.min[0]), b.res);
    const double fy = __ddiv_rn(__dsub_rn((double)c.y[i], b.min[1]), b.res);
    const double fz = __ddiv_rn(__dsub_rn((double)c.z[i], b.min[2]), b.res);
    const double lim = (double)(1u << b.depth);
    *inside = fx >= 0.0 && fy >= 0.0 && fz >= 0.0 && fx < lim && fy < lim && fz < lim;
    const uint32_t kx = (uint32_t)__double2uint_rz(fx), ky = (uint32_t)__double2uint_rz(fy), kz = (uint32_t)__double2uint_rz(fz);
    return (spread3(kx) << 2) | (spread3(ky) << 1) | spread3(kz);
}

// Also reports (unsorted != nullptr) whether the codes are NOT strictly increasing in input order, for the shortcut below.  Blocks
// overlap by one point (block b covers points b*255 .. b*255+255) so that every point finds its predecessor's code inside its own
// block -- through the neighbouring lane or shared memory -- without a divergent recomputation of the f64 divisions.
constexpr int kVoxKeyStride = 255;
// idx == nullptr: packed mode, keys[i] = code << pack_shift | i (the caller checked that both fit 64 bits)
__global__ void __launch_bounds__(256) vox_key_kernel(PtrView c, VoxBox b, uint64_t* __restrict__ keys, uint32_t* __restrict__ idx, int pack_shift,
                                                      unsigned int* __restrict__ bad, unsigned int* __restrict__ unsorted) {
    __shared__ uint64_t s_last[8];   // code of lane 31 of each warp
    const int64_t i = (int64_t)blockIdx.x * kVoxKeyStride + threadIdx.x;
    const bool live = i < c.n;
    const bool owner = live && (threadIdx.x > 0 || blockIdx.x == 0);   // thread 0 of later blocks only re-derives the previous block's last code
    uint64_t key = 0;
    if (live) {
        bool inside;
        key = vox_code(c, b, i, &inside);
        if (owner) {
            if (!inside) atomicAdd(bad, 1u);
            if (idx) { keys[i] = key; idx[i] = (uint32_t)i; }
            else keys[i] = (key << pack_shift) | (uint64_t)i;
        }
    }
    if (unsorted) {
        const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        uint64_t prev = __shfl_up_sync(0xffffffffu, key, 1);
        if (lane == 31) s_last[warp] = key;
        __syncthreads();
        if (lane == 0 && warp > 0) prev = s_last[warp - 1];
        const bool out_of_order = live && threadIdx.x > 0 && !(key > prev);
        // unsorted inputs would otherwise send one atomic per warp to the same address (measured: 2.7x slower on a 40 M-point cloud)
        if (__any_sync(0xffffffffu, out_of_order) && lane == 0 && *(volatile unsigned int*)unsorted == 0u) atomicOr(unsorted, 1u);
    }
}

__global__ void __launch_bounds__(256) vox_head_kernel(const uint64_t* __restrict__ keys, int pack_shift, int64_t n, uint32_t* __restrict__ head) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    head[i] = (i == 0 || (keys[i] >> pack_shift) != (keys[i - 1] >> pack_shift)) ? 1u : 0u;
}

// one thread per voxel: find its run [start, end) and sum sequentially in sorted (== insertion) order
__global__ void __launch_bounds__(256) vox_centroid_kernel(PtrView c, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ idx, int pack_shift,
                                                           const uint32_t* __restrict__ head, const uint32_t* __restrict__ rank, int64_t n,
                                                           DevCloud out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !head[i]) return;
    const uint64_t idx_mask = ((uint64_t)1 << pack_shift) - 1;
    uint64_t kj = keys[i];
    const uint64_t code = kj >> pack_shift;
    float sx = 0.0f, sy = 0.0f, sz = 0.0f, si = 0.0f;
    int64_t j = i;
    int cnt = 0;
    do {
        const uint32_t p = idx ? idx[j] : (uint32_t)(kj & idx_mask);
        sx = fa(sx, c.x[p]); sy = fa(sy, c.y[p]); sz = fa(sz, c.z[p]); si = fa(si, c.i[p]);
        ++cnt; ++j;
        if (j >= n) break;
        kj = keys[j];
    } while ((kj >> pack_shift) == code);
    const float fc = (float)cnt;
    const uint32_t o = rank[i];
    out.x()[o] = fd(sx, fc); out.y()[o] = fd(sy, fc); out.z()[o] = fd(sz, fc); out.i()[o] = fd(si, fc);
}

// Shortcut for inputs that are already one point per voxel in octree order (typical: the static subset of a voxelised map,
// re-voxelised at the same leaf by removeOnce, Removerter.cpp:893-896, when the removed points did not move the bounding box).
// Decided on the keys of THIS call's box, so it needs no provenance: strictly increasing codes <=> the sort is the identity and
// every run has length one, and the centroid of a single point is (0.0f + p) / 1.0f -- the same two f32 operations as below.
__global__ void __launch_bounds__(256) vox_single_kernel(PtrView c, DevCloud out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.n) return;
    out.x()[i] = fd(fa(0.0f, c.x[i]), 1.0f); out.y()[i] = fd(fa(0.0f, c.y[i]), 1.0f);
    out.z()[i] = fd(fa(0.0f, c.z[i]), 1.0f); out.i()[i] = fd(fa(0.0f, c.i[i]), 1.0f);
}
constexpr int64_t kVoxShortcutMin = 100000;   // below this the whole voxelisation is launch-bound and the extra sync does not pay

// `out` must be allocated with cap >= in.n; sets out->n
// given_box: the box of a larger cloud this view is a part of (distributed voxelisation); otherwise the box of the view itself
static int voxel_view(ltr_ctx* ctx, const PtrView& v, float leaf, DevCloud* out, const VoxBox* given_box = nullptr) {
    const int64_t n = v.n;
    if (n == 0) { out->n = 0; return LTR_OK; }
    if (!(leaf > 0.0f)) return fail(ctx, LTR_ERR_INVALID, "voxel leaf must be positive");
    if (n >= (int64_t)1 << 31) return fail(ctx, LTR_ERR_UNSUPPORTED, "cloud too large for voxel centroid");
    float mn[3], mx[3];
    if (!given_box) {
        uint32_t nonfinite = 0;
        LTR_TRY(minmax_view(ctx, v, mn, mx, &nonfinite));
        // rejected before define_box, whose cast of ceil(inf or NaN) to unsigned is undefined
        if (nonfinite) return fail(ctx, LTR_ERR_UNSUPPORTED, "%u points with non-finite coordinates", nonfinite);
    }
    const VoxBox b = given_box ? *given_box : define_box(mn, mx, leaf);
    if (b.depth > 21) return fail(ctx, LTR_ERR_UNSUPPORTED, "octree depth %d > 21 (extent/leaf too large)", b.depth);
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    const size_t kb = (size_t)n * sizeof(uint64_t), ib = (size_t)n * sizeof(uint32_t);
    // the point index rides in the low bits of the sort key when Morton code + index fit 64 bits (every cloud of the path: depth <= 12,
    // n < 2^28); the stable sort then moves 8-byte keys only and still leaves equal codes in insertion order
    int idx_bits = 1;
    while (idx_bits < 32 && ((int64_t)1 << idx_bits) < n) ++idx_bits;
    const bool packed = 3 * b.depth + idx_bits <= 64;
    const int pack_shift = packed ? idx_bits : 0;
    LTR_TRY(dev_alloc(ctx, &p, 2 * kb + (packed ? 2 : 4) * ib + 256));
    uint64_t* keys0 = (uint64_t*)p;
    uint64_t* keys1 = keys0 + n;
    uint32_t* idx0 = packed ? nullptr : (uint32_t*)(keys1 + n);
    uint32_t* idx1 = packed ? nullptr : idx0 + n;
    uint32_t* head = packed ? (uint32_t*)(keys1 + n) : idx1 + n;
    uint32_t* rank = head + n;
    unsigned int* bad = (unsigned int*)(rank + n);
    LTR_CUDA(ctx, cudaMemsetAsync(bad, 0, sizeof(unsigned int), ctx->stream));
    const int T = 256;
    const unsigned nb = (unsigned)((n + T - 1) / T);
    const bool try_shortcut = n >= kVoxShortcutMin;
    LTR_CUDA(ctx, cudaMemsetAsync(bad + 1, 0, sizeof(unsigned int), ctx->stream));
    vox_key_kernel<<<(unsigned)((n + kVoxKeyStride - 1) / kVoxKeyStride), T, 0, ctx->stream>>>(v, b, keys0, idx0, pack_shift, bad, try_shortcut ? bad + 1 : nullptr);
    LTR_LAUNCH_CHECK(ctx);
    if (try_shortcut) {
        unsigned int h[2] = {0, 1};
        LTR_CUDA(ctx, cudaMemcpyAsync(h, bad, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (h[0]) { g_p.release(); return fail(ctx, LTR_ERR_UNSUPPORTED, "%u points fall outside the octree bounding box (non-finite coordinates?)", h[0]); }
        if (!h[1]) {
            vox_single_kernel<<<nb, T, 0, ctx->stream>>>(v, *out);
            LTR_LAUNCH_CHECK(ctx);
            g_p.release();
            out->n = n;
            ctx->vox_shortcuts++;
            return LTR_OK;
        }
    }
    uint64_t* keys_s; uint32_t* idx_s;
    LTR_TRY(radix_sort_pairs(ctx, keys0, keys1, idx0, idx1, n, pack_shift, pack_shift + 3 * b.depth, &keys_s, &idx_s));
    vox_head_kernel<<<nb, T, 0, ctx->stream>>>(keys_s, pack_shift, n, head);
    LTR_LAUNCH_CHECK(ctx);
    LTR_TRY(exclusive_scan_u32(ctx, head, rank, n));
    vox_centroid_kernel<<<nb, T, 0, ctx->stream>>>(v, keys_s, idx_s, pack_shift, head, rank, n, *out);
    LTR_LAUNCH_CHECK(ctx);
    uint32_t last[2];
    unsigned int hbad = 0;
    LTR_CUDA(ctx, cudaMemcpyAsync(&last[0], rank + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaMemcpyAsync(&last[1], head + n - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaMemcpyAsync(&hbad, bad, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    g_p.release();
    if (hbad) return fail(ctx, LTR_ERR_UNSUPPORTED, "%u points fall outside the octree bounding box (non-finite coordinates?)", hbad);
    out->n = (int64_t)last[0] + last[1];
    return LTR_OK;
}

// ------------------------------------------------------------------------------------------------
// Distributed voxel centroid: octreeDownsampling (utility.cpp:204-219) of the rank-ordered CONCATENATION of every rank's local
// cloud, without ever materialising that concatenation.  The merged clouds of the path (utility.cpp:177-189 concatenates the
// keyframes in order; contiguous keyframe blocks make that the rank order) are only ever consumed through the voxeliser, and
// gathering 60 M raw points to sort them on every rank was what stopped the multi-GPU step from scaling.
//   1. global bounding box: ncclAllReduce(min / max) of the ordered-uint encoded local extrema -> the SAME VoxBox as the gathered cloud
//   2. every rank computes the Morton keys of its local points; a 4096-bin histogram of the key prefixes is all-reduced and cut
//      into `world` contiguous prefix ranges of (nearly) equal population -- a voxel never straddles a cut
//   3. one stable radix pass on the destination rank groups the local points by destination; grouped ncclSend/ncclRecv moves
//      each group to its owner, which receives them in source-rank order == global insertion order
//   4. the owner voxelises its range with the global box (stable sort + sequential f32 sums: bit-identical to the serial result)
//   5. the centroid slices (8x fewer points than the input) are all-gathered in range order == octree order.
// The rank-local work is split into the stages A-D below, which every rank runs between the collectives; voxel_distributed joins
// them with NCCL, ltr_debug_voxel_distributed with host reductions and concatenations over simulated ranks of one context.  Every
// decision that ends the call early is taken on a reduced value, so all ranks leave at the same point.
// ------------------------------------------------------------------------------------------------
constexpr int kDistHistBits = 12;
constexpr int kDistHistWords = (1 << kDistHistBits) + 1;   // prefix bins, then the points outside the box
// one rank's extrema block: [0, 3) min xyz, [3, 6) max xyz (ordered encodings), [6] points with a non-finite coordinate or
// kDistTooLarge; then the local and the global histogram (kDistHistWords each).  [0, 3) is min-reduced, [3, 7) max-reduced.
constexpr int kDistMmWords = 7;
constexpr uint32_t kDistTooLarge = 0xffffffffu;
constexpr size_t kDistMmBytes = (8 + 2 * (size_t)kDistHistWords) * sizeof(uint32_t);

// a point outside the box (counted by vox_key_kernel, and the call is rejected) has a code past the last bin: it is not binned
__global__ void __launch_bounds__(256) vox_prefix_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift, uint32_t nbins,
                                                              uint32_t* __restrict__ hist) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t b = keys[i] >> shift;
        if (b < nbins) atomicAdd(&hist[b], 1u);     // Morton-ordered or scan-ordered inputs: neighbouring threads mostly hit different bins
    }
}

struct DestCuts { uint32_t ub[16]; int world; };   // destination of prefix bin b = number of cuts ub[j] (j < world - 1) with b >= ub[j]

__global__ void __launch_bounds__(256) vox_dest_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift, DestCuts cuts, uint64_t* __restrict__ dkey,
                                                       uint32_t* __restrict__ didx) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t b = (uint32_t)(keys[i] >> shift);
    unsigned d = 0;
    for (int j = 0; j < cuts.world - 1; ++j) d += (b >= cuts.ub[j]) ? 1u : 0u;
    dkey[i] = d; didx[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) gather_points_kernel(PtrView in, const uint32_t* __restrict__ idx, DevCloud out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= in.n) return;
    const uint32_t s = idx[i];
    out.x()[i] = in.x[s]; out.y()[i] = in.y[s]; out.z()[i] = in.z[s]; out.i()[i] = in.i[s];
}

static int dist_check_args(ltr_ctx* ctx, int G, float leaf) {
    if (!(leaf > 0.0f)) return fail(ctx, LTR_ERR_INVALID, "voxel leaf must be positive");
    if (G > 16) return fail(ctx, LTR_ERR_UNSUPPORTED, "distributed voxeliser: more than 16 ranks");
    return LTR_OK;
}

// Stage A: allocates the rank's extrema block (kDistMmBytes) and enqueues its local extrema and non-finite count
static int dist_stage_extrema(ltr_ctx* ctx, const PtrView& loc, void** mm_block) {
    LTR_TRY(dev_alloc(ctx, mm_block, kDistMmBytes));
    uint32_t* d_mm = (uint32_t*)*mm_block;
    const bool too_large = loc.n >= (int64_t)1 << 31;
    const uint32_t init[kDistMmWords] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, too_large ? kDistTooLarge : 0u};
    LTR_CUDA(ctx, cudaMemcpyAsync(d_mm, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    if (loc.n > 0 && !too_large) {
        const int blocks = (int)std::min<int64_t>((loc.n + 255) / 256, (int64_t)ctx->sm_count * 8);
        minmax_kernel<<<std::max(blocks, 1), 256, 0, ctx->stream>>>(loc, d_mm, d_mm + 6);
        LTR_LAUNCH_CHECK(ctx);
    }
    return LTR_OK;
}

// From the reduced extrema block: rejects non-finite input before define_box (whose cast of ceil(inf or NaN) to unsigned is undefined)
// and before the empty test (an all-NaN cloud has no extrema), then either reports that every rank is empty or gives the global box and
// the prefix histogram's bits and shift
static int dist_decide_box(ltr_ctx* ctx, const uint32_t mm[kDistMmWords], float leaf, bool* empty, VoxBox* b, int* hb, int* shift) {
    if (mm[6] == kDistTooLarge) return fail(ctx, LTR_ERR_UNSUPPORTED, "cloud too large for voxel centroid");
    if (mm[6]) return fail(ctx, LTR_ERR_UNSUPPORTED, "points with non-finite coordinates (up to %u on one rank)", mm[6]);
    *empty = mm[0] == 0xffffffffu && mm[3] == 0u;
    if (*empty) return LTR_OK;
    float mn[3], mx[3];
    for (int d = 0; d < 3; ++d) { mn[d] = ord2f(mm[d]); mx[d] = ord2f(mm[3 + d]); }
    *b = define_box(mn, mx, leaf);
    if (b->depth > 21) return fail(ctx, LTR_ERR_UNSUPPORTED, "octree depth %d > 21 (extent/leaf too large)", b->depth);
    *hb = std::min(kDistHistBits, 3 * b->depth);
    *shift = 3 * b->depth - *hb;
    return LTR_OK;
}

// the key block of a rank with n local points: keys0 | keys1 | idx0 | idx1
struct DistKeys { uint64_t *keys0, *keys1; uint32_t *idx0, *idx1; };
static DistKeys dist_keys(void* block, int64_t n) {
    const int64_t nn = std::max<int64_t>(n, 1);
    DistKeys k;
    k.keys0 = (uint64_t*)block; k.keys1 = k.keys0 + nn;
    k.idx0 = (uint32_t*)(k.keys1 + nn); k.idx1 = k.idx0 + nn;
    return k;
}

// Stage B: allocates the key block and enqueues the local Morton keys under the global box and the local prefix histogram into
// hist[0, 2^hb), the points outside the box into hist[2^hb]; clears the global histogram after it
static int dist_stage_keys(ltr_ctx* ctx, const PtrView& loc, const VoxBox& b, int hb, int shift, uint32_t* hist, void** key_block) {
    const int64_t n = loc.n, nn = std::max<int64_t>(n, 1);
    LTR_TRY(dev_alloc(ctx, key_block, 2 * (size_t)nn * sizeof(uint64_t) + 2 * (size_t)nn * sizeof(uint32_t)));
    const DistKeys k = dist_keys(*key_block, n);
    LTR_CUDA(ctx, cudaMemsetAsync(hist, 0, 2 * (size_t)kDistHistWords * sizeof(uint32_t), ctx->stream));
    if (n > 0) {
        vox_key_kernel<<<(unsigned)((n + kVoxKeyStride - 1) / kVoxKeyStride), 256, 0, ctx->stream>>>(loc, b, k.keys0, k.idx0, 0, hist + (1 << hb), nullptr);
        LTR_LAUNCH_CHECK(ctx);
        const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 8);
        vox_prefix_hist_kernel<<<std::max(blocks, 1), 256, 0, ctx->stream>>>(k.keys0, n, shift, 1u << hb, hist);
        LTR_LAUNCH_CHECK(ctx);
    }
    return LTR_OK;
}

// Stage C, host part, from the global histogram hg (identical on every rank; hg[nbins] = points outside the box) and this rank's hl:
// the cuts, and how many of this rank's points go to each rank
static int dist_plan(ltr_ctx* ctx, const uint32_t* hl, const uint32_t* hg, int nbins, int G, DestCuts* cuts, std::vector<int64_t>* scount) {
    if (hg[nbins]) return fail(ctx, LTR_ERR_UNSUPPORTED, "%u points fall outside the octree bounding box (non-finite coordinates?)", hg[nbins]);
    uint64_t total = 0;
    for (int i = 0; i < nbins; ++i) total += hg[i];
    cuts->world = G;
    {   // cut j = first bin at which the cumulative population reaches (j + 1) / G of the total
        uint64_t cum = 0;
        int j = 0;
        for (int i = 0; i < nbins && j < G - 1; ++i) {
            cum += hg[i];
            while (j < G - 1 && cum * (uint64_t)G >= total * (uint64_t)(j + 1)) cuts->ub[j++] = (uint32_t)(i + 1);
        }
        while (j < G - 1) cuts->ub[j++] = (uint32_t)nbins;
    }
    scount->assign((size_t)G, 0);
    std::vector<uint64_t> range((size_t)G, 0);
    for (int i = 0; i < nbins; ++i) {
        int d = 0;
        for (int j = 0; j < G - 1; ++j) d += ((uint32_t)i >= cuts->ub[j]) ? 1 : 0;
        (*scount)[(size_t)d] += hl[i];
        range[(size_t)d] += hg[i];
    }
    for (int d = 0; d < G; ++d)
        if (range[(size_t)d] >= (uint64_t)1 << 31) return fail(ctx, LTR_ERR_UNSUPPORTED, "cloud too large for voxel centroid (range %d)", d);
    return LTR_OK;
}

// Stage C, device part: groups the local points by destination (stable) into `send`, segment d holding the points of range d
static int dist_stage_group(ltr_ctx* ctx, const PtrView& loc, void* key_block, int shift, const DestCuts& cuts, const DevCloud& send) {
    const int64_t n = loc.n;
    if (n == 0) return LTR_OK;
    const DistKeys k = dist_keys(key_block, n);
    vox_dest_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(k.keys0, n, shift, cuts, k.keys1, k.idx1);
    LTR_LAUNCH_CHECK(ctx);
    uint64_t* ks; uint32_t* is;
    LTR_TRY(radix_sort_pairs(ctx, k.keys1, k.keys0, k.idx1, k.idx0, n, 0, 8, &ks, &is));
    gather_points_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(loc, is, send);
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

// Stage D is voxel_view(recv, leaf, &slice, &global_box): the owner's range with the GLOBAL box.

static int voxel_distributed(ltr_ctx* ctx, int comm, const DevCloud& loc, float leaf, ltr_cloud* out_h) {
    int me = 0, G = 1;
    LTR_TRY(nccl_comm_info(ctx, comm, &me, &G));
    LTR_TRY(dist_check_args(ctx, G, leaf));
    const PtrView lv = view(loc);
    // A. global extrema and non-finite flag
    void* p_mm = nullptr;
    ScratchGuard g_mm(ctx, &p_mm);
    LTR_TRY(dist_stage_extrema(ctx, lv, &p_mm));
    uint32_t* d_mm = (uint32_t*)p_mm;
    LTR_TRY(nccl_allreduce_u32(ctx, comm, d_mm, 3, 1));
    LTR_TRY(nccl_allreduce_u32(ctx, comm, d_mm + 3, 4, 2));
    uint32_t h_mm[kDistMmWords];
    LTR_CUDA(ctx, cudaMemcpyAsync(h_mm, d_mm, sizeof(h_mm), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    bool empty = false;
    VoxBox b;
    int hb = 0, shift = 0;
    LTR_TRY(dist_decide_box(ctx, h_mm, leaf, &empty, &b, &hb, &shift));
    if (empty) { CloudOwner h; LTR_TRY(cloud_new(ctx, 0, &h)); *out_h = h.release(); return LTR_OK; }   // every rank's cloud is empty
    // B. local keys + prefix histogram, summed over the ranks
    uint32_t* d_hist_loc = d_mm + 8;
    uint32_t* d_hist_glb = d_hist_loc + kDistHistWords;
    const int nbins = 1 << hb;
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dist_stage_keys(ctx, lv, b, hb, shift, d_hist_loc, &p));
    LTR_CUDA(ctx, cudaMemcpyAsync(d_hist_glb, d_hist_loc, (size_t)(nbins + 1) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    LTR_TRY(nccl_allreduce_u32(ctx, comm, d_hist_glb, (size_t)nbins + 1, 0));
    std::vector<uint32_t> h_hist(2 * (size_t)kDistHistWords);
    LTR_CUDA(ctx, cudaMemcpyAsync(h_hist.data(), d_hist_loc, h_hist.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    // C. group the local points by destination (stable), move them to their owners
    DestCuts cuts;
    std::vector<int64_t> scount;
    LTR_TRY(dist_plan(ctx, h_hist.data(), h_hist.data() + kDistHistWords, nbins, G, &cuts, &scount));
    CloudOwner g_send, g_recv, g_slice;
    LTR_TRY(cloud_new(ctx, lv.n, &g_send));
    LTR_TRY(dist_stage_group(ctx, lv, p, shift, cuts, ctx->clouds[g_send.get()]));
    g_p.release();
    LTR_TRY(nccl_alltoallv_cloud(ctx, comm, ctx->clouds[g_send.get()], scount, &g_recv));
    g_send.reset();
    // D. my range, with the GLOBAL box
    const DevCloud recv = ctx->clouds[g_recv.get()];
    LTR_TRY(cloud_new(ctx, recv.n, &g_slice));
    DevCloud slice = ctx->clouds[g_slice.get()];
    LTR_TRY(voxel_view(ctx, view(recv), leaf, &slice, &b));
    ctx->clouds[g_slice.get()].n = slice.n;
    // slices in range order == octree order
    const ltr_cloud local[1] = {g_slice.get()};
    return ltr_nccl_allgather_clouds(ctx, comm, 1, local, out_h);
}

// The stages of voxel_distributed for `world` simulated ranks of one context: the min / max and sum all-reduces become host reductions,
// the alltoallv a concatenation of every rank's destination segment in source-rank order, the all-gather a concatenation in rank order.
static int voxel_distributed_simulated(ltr_ctx* ctx, int G, const ltr_cloud* locals, float leaf, ltr_cloud* out_h, uint32_t* cuts_out,
                                       int64_t* send_counts) {
    LTR_TRY(dist_check_args(ctx, G, leaf));
    std::vector<PtrView> lv((size_t)G);
    for (int r = 0; r < G; ++r) { DevCloud* c; LTR_TRY(cloud_get(ctx, locals[r], &c)); lv[(size_t)r] = view(*c); }
    std::vector<void*> p_mm((size_t)G, nullptr), p_keys((size_t)G, nullptr);
    std::deque<ScratchGuard> guards;
    for (int r = 0; r < G; ++r) { guards.emplace_back(ctx, &p_mm[(size_t)r]); guards.emplace_back(ctx, &p_keys[(size_t)r]); }
    // A
    uint32_t mm[kDistMmWords] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u};
    for (int r = 0; r < G; ++r) {
        LTR_TRY(dist_stage_extrema(ctx, lv[(size_t)r], &p_mm[(size_t)r]));
        uint32_t h[kDistMmWords];
        LTR_CUDA(ctx, cudaMemcpyAsync(h, p_mm[(size_t)r], sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int w = 0; w < kDistMmWords; ++w) mm[w] = w < 3 ? std::min(mm[w], h[w]) : std::max(mm[w], h[w]);
    }
    bool empty = false;
    VoxBox b;
    int hb = 0, shift = 0;
    LTR_TRY(dist_decide_box(ctx, mm, leaf, &empty, &b, &hb, &shift));
    if (cuts_out) for (int j = 0; j < G - 1; ++j) cuts_out[j] = 0;
    if (send_counts) for (int j = 0; j < G * G; ++j) send_counts[j] = 0;
    if (empty) { CloudOwner h; LTR_TRY(cloud_new(ctx, 0, &h)); *out_h = h.release(); return LTR_OK; }
    // B
    const int nbins = 1 << hb;
    std::vector<uint32_t> hl((size_t)G * kDistHistWords), hg((size_t)kDistHistWords, 0u);
    for (int r = 0; r < G; ++r) {
        uint32_t* hist = (uint32_t*)p_mm[(size_t)r] + 8;
        LTR_TRY(dist_stage_keys(ctx, lv[(size_t)r], b, hb, shift, hist, &p_keys[(size_t)r]));
        LTR_CUDA(ctx, cudaMemcpyAsync(&hl[(size_t)r * kDistHistWords], hist, kDistHistWords * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    }
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int r = 0; r < G; ++r)
        for (int i = 0; i <= nbins; ++i) hg[(size_t)i] += hl[(size_t)r * kDistHistWords + i];
    // C
    DestCuts cuts;
    std::vector<std::vector<int64_t>> scount((size_t)G);
    for (int r = 0; r < G; ++r) LTR_TRY(dist_plan(ctx, &hl[(size_t)r * kDistHistWords], hg.data(), nbins, G, &cuts, &scount[(size_t)r]));
    std::deque<CloudOwner> send, recv, slice;
    for (int r = 0; r < G; ++r) {
        send.emplace_back();
        LTR_TRY(cloud_new(ctx, lv[(size_t)r].n, &send.back()));
        LTR_TRY(dist_stage_group(ctx, lv[(size_t)r], p_keys[(size_t)r], shift, cuts, ctx->clouds[send.back().get()]));
    }
    guards.clear();
    for (int d = 0; d < G; ++d) {
        int64_t m = 0;
        for (int r = 0; r < G; ++r) m += scount[(size_t)r][(size_t)d];
        recv.emplace_back();
        LTR_TRY(cloud_new(ctx, m, &recv.back()));
        const DevCloud dst = ctx->clouds[recv.back().get()];
        int64_t at = 0;
        for (int r = 0; r < G; ++r) {
            const DevCloud src = ctx->clouds[send[(size_t)r].get()];
            int64_t from = 0;
            for (int e = 0; e < d; ++e) from += scount[(size_t)r][(size_t)e];
            const int64_t k = scount[(size_t)r][(size_t)d];
            if (k > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(dst.base + at, (size_t)dst.cap * 4, src.base + from, (size_t)src.cap * 4, (size_t)k * 4, 4,
                                                       cudaMemcpyDeviceToDevice, ctx->stream));
            at += k;
        }
    }
    send.clear();
    // D
    int64_t total = 0;
    for (int d = 0; d < G; ++d) {
        const DevCloud rc = ctx->clouds[recv[(size_t)d].get()];
        slice.emplace_back();
        LTR_TRY(cloud_new(ctx, rc.n, &slice.back()));
        DevCloud s = ctx->clouds[slice.back().get()];
        LTR_TRY(voxel_view(ctx, view(rc), leaf, &s, &b));
        ctx->clouds[slice.back().get()].n = s.n;
        total += s.n;
    }
    CloudOwner g_out;
    LTR_TRY(cloud_new(ctx, total, &g_out));
    const DevCloud o = ctx->clouds[g_out.get()];
    int64_t at = 0;
    for (int d = 0; d < G; ++d) {
        const DevCloud s = ctx->clouds[slice[(size_t)d].get()];
        if (s.n > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(o.base + at, (size_t)o.cap * 4, s.base, (size_t)s.cap * 4, (size_t)s.n * 4, 4,
                                                     cudaMemcpyDeviceToDevice, ctx->stream));
        at += s.n;
    }
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (cuts_out) for (int j = 0; j < G - 1; ++j) cuts_out[j] = cuts.ub[j];
    if (send_counts) for (int r = 0; r < G; ++r) for (int d = 0; d < G; ++d) send_counts[r * G + d] = scount[(size_t)r][(size_t)d];
    *out_h = g_out.release();
    return LTR_OK;
}

// ------------------------------------------------------------------------------------------------
// Frame changes of scan sets: local2global of the points [base, base + n) (utility.cpp:164-165), and global2local back (utility.cpp:198-199)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) scans_to_global_kernel(PtrView in, const int64_t* __restrict__ off, int K, int64_t base, int64_t n,
                                                              const double* __restrict__ poses, const double* __restrict__ ext, int order,
                                                              float* __restrict__ ox, float* __restrict__ oy, float* __restrict__ oz,
                                                              float* __restrict__ oi, const float* __restrict__ T16,
                                                              const uint8_t* __restrict__ accept) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int64_t i = base + t;
    const int k = find_kf(off, K, i);
    float x = in.x[i], y = in.y[i], z = in.z[i];
    scan_to_global(poses + (size_t)k * 24 + 12, ext, order, &x, &y, &z);
    refine_point(T16, accept, k, &x, &y, &z);
    ox[t] = x; oy[t] = y; oz[t] = z;
    if (oi) oi[t] = in.i[i];
}

__global__ void __launch_bounds__(256) global_to_scans_kernel(const float* __restrict__ gx, const float* __restrict__ gy, const float* __restrict__ gz,
                                                              const int64_t* __restrict__ off, int K, int64_t base, int64_t n,
                                                              const double* __restrict__ poses, const double* __restrict__ ext, int order,
                                                              DevCloud out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int64_t i = base + t;
    const int k = find_kf(off, K, i);
    map_to_sensor(poses + (size_t)k * 24, ext, ext == nullptr, order, gx[t], gy[t], gz[t], &out.x()[i], &out.y()[i], &out.z()[i]);
}

int scans_to_global(ltr_ctx* ctx, const DevScanSet& scans, int64_t base, int64_t n, const double* poses, const double* ext, float* ox,
                    float* oy, float* oz, float* oi, const float* T16, const uint8_t* accept) {
    if (n == 0) return LTR_OK;
    scans_to_global_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(view(scans.pts), scans.d_off, scans.K, base, n, poses, ext,
                                                                                ctx->cfg.transform_order, ox, oy, oz, oi, T16, accept);
    LTR_LAUNCH_CHECK(ctx);
    return LTR_OK;
}

int upload_refinement(ltr_ctx* ctx, int K, const float* T16, const uint8_t* accepted, float* dT, uint8_t* dacc) {
    std::vector<uint8_t> acc((size_t)K);
    for (int j = 0; j < K; ++j) acc[j] = accepted[j] ? 1 : 0;
    LTR_CUDA(ctx, cudaMemcpyAsync(dT, T16, (size_t)K * 64, cudaMemcpyHostToDevice, ctx->stream));
    LTR_CUDA(ctx, cudaMemcpyAsync(dacc, acc.data(), (size_t)K, cudaMemcpyHostToDevice, ctx->stream));
    return LTR_OK;
}

int ScanSplit::init() {
    return scans_.pts.n > 0 ? dev_alloc(ctx_, (void**)&flags, (size_t)scans_.pts.n) : LTR_OK;
}

int ScanSplit::relocalise(int64_t base, int64_t n, const float* gx, const float* gy, const float* gz) {
    if (n == 0) return LTR_OK;
    if (reloc_.get() < 0) {
        LTR_TRY(cloud_new(ctx_, scans_.pts.n, &reloc_));
        LTR_CUDA(ctx_, cudaMemcpyAsync(ctx_->clouds[reloc_.get()].i(), scans_.pts.i(), (size_t)scans_.pts.n * sizeof(float), cudaMemcpyDeviceToDevice,
                                       ctx_->stream));
    }
    global_to_scans_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx_->stream>>>(gx, gy, gz, scans_.d_off, scans_.K, base, n, poses_,
        ctx_->ext_identity ? nullptr : ctx_->d_ext, ctx_->cfg.transform_order, ctx_->clouds[reloc_.get()]);
    LTR_LAUNCH_CHECK(ctx_);
    return LTR_OK;
}

int ScanSplit::finish(ltr_scanset* out0, ltr_scanset* out1) {
    if (scans_.pts.n == 0) {
        const std::vector<int64_t> off((size_t)scans_.K + 1, 0);
        ScanSetOwner o0, o1;
        if (out0) LTR_TRY(scanset_new(ctx_, off, &o0));
        if (out1) LTR_TRY(scanset_new(ctx_, off, &o1));
        if (out0) *out0 = o0.release();
        if (out1) *out1 = o1.release();
        return LTR_OK;
    }
    DevScanSet set = scans_;
    set.pts = ctx_->clouds[reloc_.get()];
    return split_scanset_by_flag(ctx_, set, flags, out0, out1);
}

int64_t env_points(const char* name, int64_t def, int64_t hi) {
    if (const char* e = std::getenv(name)) if (*e) return std::min<int64_t>(std::max<int64_t>(std::atoll(e), 1), hi);
    return def;
}

std::vector<int> plan_keyframe_chunks(const std::vector<int64_t>& off, int64_t cap, int max_kf, int64_t* max_points) {
    const int K = (int)off.size() - 1;
    std::vector<int> cut{0};
    *max_points = 0;
    for (int kf = 0; kf < K;) {
        int e = kf + 1;
        while (e < K && e - kf < max_kf && off[e + 1] - off[kf] <= cap) ++e;
        cut.push_back(e);
        *max_points = std::max(*max_points, off[e] - off[kf]);
        kf = e;
    }
    return cut;
}

// precleaningKeyframes (Session.cpp:506-533)
__global__ void __launch_bounds__(256) preclean_flag_kernel(PtrView in, float radius, uint8_t* __restrict__ drop) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= in.n) return;
    const float x = in.x[i], y = in.y[i], z = in.z[i];
    const float r = __fsqrt_rn(fa(fa(fm(x, x), fm(y, y)), fm(z, z)));
    drop[i] = (r < radius && (double)z < 0.5 && -0.5 < (double)z) ? 1 : 0;
}

__global__ void segment_count_kernel(const uint8_t* __restrict__ flags, const int64_t* __restrict__ off, int K, unsigned long long* __restrict__ cnt) {
    const int k = blockIdx.x;
    if (k >= K) return;
    unsigned long long c = 0;
    for (int64_t i = off[k] + threadIdx.x; i < off[k + 1]; i += blockDim.x) c += flags[i] ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&cnt[k], c);
}

// per-keyframe counts of set flags -> host vector
int segment_counts(ltr_ctx* ctx, const uint8_t* flags, const DevScanSet& s, std::vector<int64_t>* counts) {
    counts->assign((size_t)s.K, 0);
    if (s.K == 0) return LTR_OK;
    void* p = nullptr;
    ScratchGuard g_p(ctx, &p);
    LTR_TRY(dev_alloc(ctx, &p, (size_t)s.K * sizeof(unsigned long long)));
    LTR_CUDA(ctx, cudaMemsetAsync(p, 0, (size_t)s.K * sizeof(unsigned long long), ctx->stream));
    segment_count_kernel<<<s.K, 256, 0, ctx->stream>>>(flags, s.d_off, s.K, (unsigned long long*)p);
    LTR_LAUNCH_CHECK(ctx);
    std::vector<unsigned long long> h((size_t)s.K);
    LTR_CUDA(ctx, cudaMemcpyAsync(h.data(), p, (size_t)s.K * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    g_p.release();
    for (int k = 0; k < s.K; ++k) (*counts)[k] = (int64_t)h[k];
    return LTR_OK;
}

// Splits a scanset by per-point flags into (unflagged, flagged) scansets, order preserved inside each keyframe.
int split_scanset_by_flag(ltr_ctx* ctx, const DevScanSet& in_ref, const uint8_t* flags, ltr_scanset* out_unflagged, ltr_scanset* out_flagged) {
    const DevScanSet in = in_ref;  // copy: the handle table may be reallocated by scanset_new
    std::vector<int64_t> cnt;
    LTR_TRY(segment_counts(ctx, flags, in, &cnt));
    std::vector<int64_t> off0((size_t)in.K + 1, 0), off1((size_t)in.K + 1, 0);
    for (int k = 0; k < in.K; ++k) {
        off1[k + 1] = off1[k] + cnt[k];
        off0[k + 1] = off0[k] + (in.h_off[k + 1] - in.h_off[k]) - cnt[k];
    }
    ScanSetOwner h0, h1;   // an output the caller does not take is freed on return
    const DevCloud src = in.pts;  // copy: the table may be reallocated by scanset_new
    LTR_TRY(scanset_new(ctx, off0, &h0));
    LTR_TRY(scanset_new(ctx, off1, &h1));
    // a global stable partition keeps keyframe order, so it lands exactly at the per-keyframe offsets
    DevCloud o0 = ctx->scansets[h0.get()].pts, o1 = ctx->scansets[h1.get()].pts;
    if (src.n > 0) {
        // outputs may be smaller than src.n in capacity only by construction of sizes: they are exact
        int64_t nf = 0;
        LTR_TRY(stable_partition_by_flag(ctx, src, flags, &nf, &o0, &o1));
        if (nf != off1[in.K]) return fail(ctx, LTR_ERR_CUDA, "internal: partition count mismatch");
    }
    if (out_unflagged) *out_unflagged = h0.release();
    if (out_flagged) *out_flagged = h1.release();
    return LTR_OK;
}

}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_voxel_centroid(ltr_ctx* ctx, ltr_cloud in, float leaf, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_voxel_centroid");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevCloud* c;
    LTR_TRY(cloud_get(ctx, in, &c));
    const DevCloud src = *c;
    CloudOwner h;
    LTR_TRY(cloud_new(ctx, src.n, &h));
    DevCloud o = ctx->clouds[h.get()];
    LTR_TRY(voxel_view(ctx, view(src), leaf, &o));
    ctx->clouds[h.get()].n = o.n;
    *out = h.release();
    return LTR_OK;
}

int ltr_nccl_voxel_centroid_merged(ltr_ctx* ctx, int32_t comm, ltr_cloud local, float leaf, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_nccl_voxel_centroid_merged");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevCloud* c;
    LTR_TRY(cloud_get(ctx, local, &c));
    const DevCloud loc = *c;
    return voxel_distributed(ctx, comm, loc, leaf, out);
}

int ltr_debug_voxel_distributed(ltr_ctx* ctx, int32_t world, const ltr_cloud* locals, float leaf, ltr_cloud* out, uint32_t* cuts,
                                int64_t* send_counts) {
    ApiTrace tr__(ctx, "ltr_debug_voxel_distributed");
    if (!ctx || !out || !locals || world < 1) return fail(ctx, LTR_ERR_INVALID, "bad argument");
    return voxel_distributed_simulated(ctx, world, locals, leaf, out, cuts, send_counts);
}

int ltr_voxel_centroid_per_keyframe(ltr_ctx* ctx, ltr_scanset in, float leaf, ltr_scanset* out) {
    ApiTrace tr__(ctx, "ltr_voxel_centroid_per_keyframe");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevScanSet* s;
    LTR_TRY(scanset_get(ctx, in, &s));
    const DevCloud src = s->pts;
    const std::vector<int64_t> off = s->h_off;
    const int K = s->K;
    // worst case every point survives: voxelise into a scratch of the input layout, then compact
    CloudOwner scratch;
    LTR_TRY(cloud_new(ctx, src.n, &scratch));
    const DevCloud sc = ctx->clouds[scratch.get()];
    std::vector<int64_t> noff((size_t)K + 1, 0);
    for (int k = 0; k < K; ++k) {
        PtrView v{src.x() + off[k], src.y() + off[k], src.z() + off[k], src.i() + off[k], off[k + 1] - off[k]};
        DevCloud o = sc;
        o.base = sc.base + off[k];  // component stride stays sc.cap
        LTR_TRY(voxel_view(ctx, v, leaf, &o));
        noff[k + 1] = noff[k] + o.n;
    }
    ScanSetOwner h;
    LTR_TRY(scanset_new(ctx, noff, &h));
    DevCloud& d = ctx->scansets[h.get()].pts;
    for (int k = 0; k < K; ++k) {
        const int64_t m = noff[k + 1] - noff[k];
        if (m > 0) LTR_CUDA(ctx, cudaMemcpy2DAsync(d.base + noff[k], (size_t)d.cap * 4, sc.base + off[k], (size_t)sc.cap * 4, (size_t)m * 4, 4, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    *out = h.release();
    return LTR_OK;
}

int ltr_merge_scans_global(ltr_ctx* ctx, ltr_scanset scans, ltr_poses poses, ltr_cloud* out) {
    ApiTrace tr__(ctx, "ltr_merge_scans_global");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevScanSet* s;
    DevPoses* p;
    LTR_TRY(scanset_get(ctx, scans, &s));
    LTR_TRY(poses_get(ctx, poses, &p));
    if (p->K != s->K) return fail(ctx, LTR_ERR_INVALID, "pose count %d != keyframe count %d (Session.cpp:117)", p->K, s->K);
    const DevScanSet ss = *s;
    const DevPoses pp = *p;
    CloudOwner h;
    LTR_TRY(cloud_new(ctx, ss.pts.n, &h));
    // mergeScansWithinGlobalCoordUtil (utility.cpp:170-192): lidar2base, then the pose
    const DevCloud o = ctx->clouds[h.get()];
    LTR_TRY(scans_to_global(ctx, ss, 0, ss.pts.n, pp.d, ctx->ext_identity ? nullptr : ctx->d_ext + 12, o.x(), o.y(), o.z(), o.i()));
    *out = h.release();
    return LTR_OK;
}

int ltr_preclean(ltr_ctx* ctx, ltr_scanset scans, float radius, ltr_scanset* out) {
    ApiTrace tr__(ctx, "ltr_preclean");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevScanSet* s;
    LTR_TRY(scanset_get(ctx, scans, &s));
    const DevScanSet ss = *s;
    void* drop = nullptr;
    ScratchGuard g_drop(ctx, &drop);
    LTR_TRY(dev_alloc(ctx, &drop, (size_t)std::max<int64_t>(ss.pts.n, 1)));
    if (ss.pts.n > 0) {
        const int T = 256;
        preclean_flag_kernel<<<(unsigned)((ss.pts.n + T - 1) / T), T, 0, ctx->stream>>>(view(ss.pts), radius, (uint8_t*)drop);
        LTR_LAUNCH_CHECK(ctx);
    }
    return split_scanset_by_flag(ctx, ss, (const uint8_t*)drop, out, nullptr);
}

int ltr_flags_device_ptr(ltr_ctx* ctx, ltr_cloud map, uint8_t** flags, int64_t* n) {
    ApiTrace tr__(ctx, "ltr_flags_device_ptr");
    DevCloud* c;
    LTR_TRY(cloud_get(ctx, map, &c));
    LTR_TRY(cloud_ensure_flags(ctx, c));
    if (flags) *flags = c->flags;
    if (n) *n = c->n;
    return LTR_OK;
}
int ltr_flags_download(ltr_ctx* ctx, ltr_cloud map, uint8_t* flags, int64_t capacity) {
    ApiTrace tr__(ctx, "ltr_flags_download");
    DevCloud* c;
    LTR_TRY(cloud_get(ctx, map, &c));
    LTR_TRY(cloud_ensure_flags(ctx, c));
    if (capacity < c->n) return fail(ctx, LTR_ERR_INVALID, "flag buffer too small");
    if (c->n > 0) LTR_CUDA(ctx, cudaMemcpyAsync(flags, c->flags, (size_t)c->n, cudaMemcpyDeviceToHost, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}
int ltr_flags_upload(ltr_ctx* ctx, ltr_cloud map, const uint8_t* flags, int64_t n) {
    ApiTrace tr__(ctx, "ltr_flags_upload");
    DevCloud* c;
    LTR_TRY(cloud_get(ctx, map, &c));
    if (n != c->n) return fail(ctx, LTR_ERR_INVALID, "flag count %lld != map size %lld", (long long)n, (long long)c->n);
    LTR_TRY(cloud_ensure_flags(ctx, c));
    if (n > 0) LTR_CUDA(ctx, cudaMemcpyAsync(c->flags, flags, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return LTR_OK;
}

int ltr_apply_partition(ltr_ctx* ctx, ltr_cloud map, ltr_cloud* out_static, ltr_cloud* out_dynamic) {
    ApiTrace tr__(ctx, "ltr_apply_partition");
    if (!ctx || !out_static || !out_dynamic) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevCloud* c;
    LTR_TRY(cloud_get(ctx, map, &c));
    // getStaticIdxFromDynamicIdx builds linspace<int>(0, N, N) (utility.h:158-167): integer step N/(N-1) is 1 only for
    // N >= 3; N == 1 divides by zero and N == 2 indexes out of range in the reference.
    if (c->n == 1 || c->n == 2) return fail(ctx, LTR_ERR_UNSUPPORTED, "maps of 1 or 2 points hit undefined behaviour in the reference (utility.h:158-167)");
    LTR_TRY(cloud_ensure_flags(ctx, c));
    const DevCloud src = *c;
    CloudOwner st, dy;
    LTR_TRY(cloud_new(ctx, src.n, &st));
    LTR_TRY(cloud_new(ctx, src.n, &dy));
    DevCloud o0 = ctx->clouds[st.get()], o1 = ctx->clouds[dy.get()];
    int64_t nf = 0;
    LTR_TRY(stable_partition_by_flag(ctx, src, src.flags, &nf, &o0, &o1));
    ctx->clouds[st.get()].n = o0.n;
    ctx->clouds[dy.get()].n = o1.n;
    *out_static = st.release();
    *out_dynamic = dy.release();
    return LTR_OK;
}

}  // extern "C"
