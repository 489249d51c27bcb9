// Load-time pcl::VoxelGrid (Session::loadKeyframes, Session.cpp:284-289) on the device, byte-identical to its restatement
// voxel_grid_span in host/io.cpp: same overflow exit, same f32 arithmetic, same x86-64 conversions of out-of-range / NaN values,
// and the same permutation of the (voxel index, point index) entries as libstdc++'s std::sort -- an introsort, NOT stable -- since
// the order of equal-index entries fixes the f32 summation order of every centroid.
//
// One CTA per scan runs the whole filter: bounding box + overflow decision, keys, introsort emulation, centroids.
//  - Segments longer than kVgSmall are partitioned by the whole CTA.  __unguarded_partition with pivot p (moved to `first` by
//    __move_median_to_first) swaps L[t] and R[t] for as long as L[t] < R[t], where L are the ascending positions of
//    [first + 1, last) holding a value >= p and R the descending positions holding a value <= p; with m such swaps it returns
//    min(L[m], R[m - 1]).  Prefix counts over the segment give every L[t] / R[t] and m directly.
//  - Shorter segments are finished by one thread each with a literal transcription of __introsort_loop (same remaining depth).
//  - A segment that reaches the depth limit gets __partial_sort(first, last, last) = make_heap + sort_heap, by one thread.
//  - __final_insertion_sort only moves an element past strictly greater ones and every segment is already partitioned against its
//    neighbours, so it equals a stable insertion sort of each leaf segment (<= 16 entries) on its own; leaves are sorted where they
//    are produced.
// tests/test_voxel_grid_sort_model.py checks these equivalences against a transcription of libstdc++ and the host library.
#include "ltr_internal.cuh"
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>

namespace ltr {

constexpr int kVgThreads = 256;
constexpr int kVgWarps = kVgThreads / 32;
constexpr uint32_t kVgSmall = 1024;          // segments at most this long are sorted by one thread
constexpr uint32_t kVgThreshold = 16;        // libstdc++ _S_threshold
constexpr int kVgStack = 128;                // CTA segment stack (LIFO: at most one entry per depth level, depth <= 62)
constexpr int64_t kVgChunkPoints = (int64_t)64 << 20;   // points per launch: bounds the 24 B/point sort scratch to 1.5 GiB

// Test knob: LTR_VOXEL_GRID_CHUNK_POINTS=n (clamped to [1, kVgChunkPoints]; unset or empty: kVgChunkPoints) takes the place of
// kVgChunkPoints in voxel_grid_run, so that tests can split small inputs into many launches and check the scratch indexing relative to
// each launch's first scan.

// x86-64 cvttss2si: NaN and out-of-range values give the "integer indefinite" 0x80000000 (CUDA saturates, and NaN -> 0)
__device__ __forceinline__ int32_t x86_f2i32(float f) {
    return (f >= -2147483648.0f && f < 2147483648.0f) ? (int32_t)f : INT32_MIN;
}
__device__ __forceinline__ int64_t x86_f2i64(float f) {
    return (f >= -9223372036854775808.0f && f < 9223372036854775808.0f) ? (int64_t)f : INT64_MIN;
}

// x86-64 SSE NaN results: a NaN operand comes through quieted (the first one if both are NaN -- the accumulator of `s += v`), an
// invalid operation (inf - inf, 0 / 0) gives the default NaN 0xffc00000.  CUDA returns the canonical 0x7fffffff for all of these.
__device__ __forceinline__ float x86_nan_in(float a, float b, bool* hit) {
    *hit = true;
    if (isnan(a)) return __uint_as_float(__float_as_uint(a) | 0x00400000u);
    if (isnan(b)) return __uint_as_float(__float_as_uint(b) | 0x00400000u);
    *hit = false;
    return 0.0f;
}
__device__ __forceinline__ float x86_add(float a, float b) {
    bool hit;
    const float q = x86_nan_in(a, b, &hit);
    if (hit) return q;
    const float r = __fadd_rn(a, b);
    return isnan(r) ? __uint_as_float(0xffc00000u) : r;
}
__device__ __forceinline__ float x86_div(float a, float b) {
    bool hit;
    const float q = x86_nan_in(a, b, &hit);
    if (hit) return q;
    const float r = __fdiv_rn(a, b);
    return isnan(r) ? __uint_as_float(0xffc00000u) : r;
}

// entry = voxel index (high 32 bits) | scan-relative point index (low 32 bits); std::less compares the index only
__device__ __forceinline__ uint32_t vkey(uint64_t e) { return (uint32_t)(e >> 32); }
__device__ __forceinline__ void vswap(uint64_t* a, int64_t i, int64_t j) { const uint64_t t = a[i]; a[i] = a[j]; a[j] = t; }

// std::__move_median_to_first(result, a, b, c)
__device__ __forceinline__ void vg_move_median_to_first(uint64_t* e, int64_t r, int64_t a, int64_t b, int64_t c) {
    const uint32_t ka = vkey(e[a]), kb = vkey(e[b]), kc = vkey(e[c]);
    int64_t s;
    if (ka < kb) s = kb < kc ? b : (ka < kc ? c : a);
    else s = ka < kc ? a : (kb < kc ? c : b);
    vswap(e, r, s);
}

// std::__adjust_heap (with its trailing __push_heap) on e[0, len)
__device__ __forceinline__ void vg_adjust_heap(uint64_t* e, int64_t hole, int64_t len, uint64_t v) {
    const int64_t top = hole;
    int64_t c = hole;
    while (c < (len - 1) / 2) {
        c = 2 * (c + 1);
        if (vkey(e[c]) < vkey(e[c - 1])) c--;
        e[hole] = e[c];
        hole = c;
    }
    if ((len & 1) == 0 && c == (len - 2) / 2) {
        c = 2 * (c + 1);
        e[hole] = e[c - 1];
        hole = c - 1;
    }
    int64_t parent = (hole - 1) / 2;
    while (hole > top && vkey(e[parent]) < vkey(v)) {
        e[hole] = e[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    e[hole] = v;
}

// std::__partial_sort(first, last, last): __make_heap, then __sort_heap
__device__ __forceinline__ void vg_heap_sort(uint64_t* e, int64_t len) {
    if (len >= 2)
        for (int64_t parent = (len - 2) / 2;; --parent) {
            vg_adjust_heap(e, parent, len, e[parent]);
            if (parent == 0) break;
        }
    while (len > 1) {
        --len;
        const uint64_t v = e[len];
        e[len] = e[0];
        vg_adjust_heap(e, 0, len, v);
    }
}

// stable insertion sort of one leaf segment (what __final_insertion_sort does to it)
__device__ __forceinline__ void vg_insertion_sort(uint64_t* e, int64_t len) {
    for (int64_t i = 1; i < len; ++i) {
        const uint64_t v = e[i];
        int64_t j = i;
        while (j > 0 && vkey(v) < vkey(e[j - 1])) { e[j] = e[j - 1]; --j; }
        e[j] = v;
    }
}

// segment descriptor: first << 32 | len << 8 | depth (len < 2^24, depth <= 62)
__device__ __forceinline__ uint64_t vg_seg(uint32_t f, uint32_t len, int d) { return ((uint64_t)f << 32) | ((uint64_t)len << 8) | (uint64_t)d; }

// std::__introsort_loop on e[f, l) with depth budget d, leaves finished by vg_insertion_sort (one thread)
__device__ __forceinline__ void vg_introsort_seq(uint64_t* e, uint32_t f, uint32_t l, int d) {
    uint64_t stk[64];   // vg_seg(first, len, depth); one entry per depth level
    int sp = 0;
    while (true) {
        bool heaped = false;
        while (l - f > kVgThreshold) {
            if (d == 0) { vg_heap_sort(e + f, l - f); heaped = true; break; }
            --d;
            vg_move_median_to_first(e, f, f + 1, f + (l - f) / 2, l - 1);
            // std::__unguarded_partition(first + 1, last, first)
            const uint32_t pk = vkey(e[f]);
            uint32_t a = f + 1, b = l;
            while (true) {
                while (vkey(e[a]) < pk) ++a;
                --b;
                while (pk < vkey(e[b])) --b;
                if (!(a < b)) break;
                vswap(e, a, b);
                ++a;
            }
            stk[sp++] = vg_seg(a, l - a, d);            // __introsort_loop(cut, last, depth_limit)
            l = a;                                       // last = cut
        }
        if (!heaped) vg_insertion_sort(e + f, l - f);
        if (sp == 0) return;
        const uint64_t g = stk[--sp];
        f = (uint32_t)(g >> 32); l = f + ((uint32_t)(g >> 8) & 0xffffffu); d = (int)(g & 0xffu);
    }
}

struct VgArgs {
    PtrView src;             // the whole input scan set
    const int64_t* off;      // its K+1 offsets
    int k0;                  // first scan of this launch
    int64_t base;            // off[k0]: scratch is indexed relative to it
    float leaf;
    uint64_t* ent;           // entries, one per point
    uint32_t* posL;          // L[t] / R[t] of the segment being partitioned
    uint32_t* posR;
    uint64_t* segs;          // short segments left for single threads: first << 32 | len << 8 | depth
    DevCloud sc;             // centroids of scan k at sc[off[k] ...]
    int64_t* cnt;            // per scan: output points
    int32_t* status;         // per scan: 0 filtered, 1 overflow exit (returned unchanged), 2 empty
};

__global__ void __launch_bounds__(kVgThreads) voxel_grid_kernel(VgArgs A) {
    __shared__ float s_mn[kVgWarps][3], s_mx[kVgWarps][3];
    __shared__ int s_pass;
    __shared__ float s_inv, s_minb[3];
    __shared__ int32_t s_mul[3];
    __shared__ uint32_t s_f[kVgStack], s_l[kVgStack];
    __shared__ int s_d[kVgStack];
    __shared__ int s_sp;
    __shared__ uint32_t s_nsmall, s_cf, s_cl, s_pk, s_totR, s_m;
    __shared__ int s_cd;
    __shared__ uint32_t s_wa[kVgWarps], s_wb[kVgWarps];

    const int k = A.k0 + blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t o = A.off[k];
    const uint32_t n = (uint32_t)(A.off[k + 1] - o);
    const float* X = A.src.x + o; const float* Y = A.src.y + o; const float* Z = A.src.z + o; const float* I = A.src.i + o;
    uint64_t* e = A.ent + (o - A.base);
    uint32_t* posL = A.posL + (o - A.base);
    uint32_t* posR = A.posR + (o - A.base);
    uint64_t* segs = A.segs + (o - A.base);
    const uint32_t lt_mask = (1u << lane) - 1u;

    if (n == 0) {
        if (tid == 0) { A.cnt[k] = 0; A.status[k] = 2; }
        return;
    }
    // ---- 1. bounding box: std::min / std::max seeded with +-FLT_MAX skip NaN
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
    for (uint32_t i = tid; i < n; i += kVgThreads) {
        const float p[3] = {X[i], Y[i], Z[i]};
        for (int d = 0; d < 3; ++d) { mn[d] = p[d] < mn[d] ? p[d] : mn[d]; mx[d] = mx[d] < p[d] ? p[d] : mx[d]; }
    }
    for (int d = 0; d < 3; ++d)
        for (int s = 16; s > 0; s >>= 1) {
            const float a = __shfl_xor_sync(0xffffffffu, mn[d], s), b = __shfl_xor_sync(0xffffffffu, mx[d], s);
            mn[d] = a < mn[d] ? a : mn[d];
            mx[d] = mx[d] < b ? b : mx[d];
        }
    if (lane == 0) for (int d = 0; d < 3; ++d) { s_mn[warp][d] = mn[d]; s_mx[warp][d] = mx[d]; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kVgWarps; ++w)
            for (int d = 0; d < 3; ++d) { mn[d] = s_mn[w][d] < mn[d] ? s_mn[w][d] : mn[d]; mx[d] = mx[d] < s_mx[w][d] ? s_mx[w][d] : mx[d]; }
        const float inv = __fdiv_rn(1.0f, A.leaf);
        uint64_t prod = 1;   // int64 product of the three extents, wrapping as on x86-64
        for (int d = 0; d < 3; ++d) prod *= (uint64_t)(x86_f2i64(__fmul_rn(__fsub_rn(mx[d], mn[d]), inv)) + 1);
        const int pass = (int64_t)prod > (int64_t)INT32_MAX ? 1 : 0;
        uint32_t div[3];
        for (int d = 0; d < 3; ++d) {
            const int32_t lo = x86_f2i32(floorf(__fmul_rn(mn[d], inv))), hi = x86_f2i32(floorf(__fmul_rn(mx[d], inv)));
            div[d] = (uint32_t)hi - (uint32_t)lo + 1u;
            s_minb[d] = __int2float_rn(lo);
        }
        s_mul[0] = 1; s_mul[1] = (int32_t)div[0]; s_mul[2] = (int32_t)(div[0] * div[1]);
        s_inv = inv;
        s_pass = pass;
        A.status[k] = pass;
        if (pass) A.cnt[k] = n;
        s_sp = 0; s_nsmall = 0;
        const int depth = 2 * (31 - __clz((int)n));   // 2 * std::__lg(n)
        if (n > kVgSmall) { s_f[0] = 0; s_l[0] = n; s_d[0] = depth; s_sp = 1; }
        else if (n > 1) { segs[0] = vg_seg(0, n, depth); s_nsmall = 1; }
    }
    __syncthreads();
    if (s_pass) return;   // output = *input_: copied by the compaction kernel
    // ---- 2. keys (int32 arithmetic wraps as the host's)
    {
        const float inv = s_inv;
        const float b0 = s_minb[0], b1 = s_minb[1], b2 = s_minb[2];
        const uint32_t m1 = (uint32_t)s_mul[1], m2 = (uint32_t)s_mul[2];
        for (uint32_t i = tid; i < n; i += kVgThreads) {
            const uint32_t i0 = (uint32_t)x86_f2i32(__fsub_rn(floorf(__fmul_rn(X[i], inv)), b0));
            const uint32_t i1 = (uint32_t)x86_f2i32(__fsub_rn(floorf(__fmul_rn(Y[i], inv)), b1));
            const uint32_t i2 = (uint32_t)x86_f2i32(__fsub_rn(floorf(__fmul_rn(Z[i], inv)), b2));
            e[i] = ((uint64_t)(i0 + i1 * m1 + i2 * m2) << 32) | i;
        }
    }
    __syncthreads();
    // ---- 3a. long segments: one CTA-wide partition at a time
    while (true) {
        if (tid == 0) {
            if (s_sp > 0) {
                --s_sp;
                s_cf = s_f[s_sp]; s_cl = s_l[s_sp]; s_cd = s_d[s_sp];
                if (s_cd > 0) {
                    vg_move_median_to_first(e, s_cf, s_cf + 1, s_cf + (s_cl - s_cf) / 2, s_cl - 1);
                    s_pk = vkey(e[s_cf]);
                }
            } else s_cd = -1;
            s_totR = 0; s_m = 0;
        }
        __syncthreads();
        const int d = s_cd;
        if (d < 0) break;
        const uint32_t f = s_cf, l = s_cl;
        if (d == 0) {   // depth limit reached (adversarial inputs only)
            if (tid == 0) vg_heap_sort(e + f, l - f);
            __syncthreads();
            continue;
        }
        const uint32_t pk = s_pk;
        // pass 1: |R|
        uint32_t c = 0;
        for (uint32_t i = f + 1 + tid; i < l; i += kVgThreads) c += vkey(e[i]) <= pk ? 1u : 0u;
        for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
        if (lane == 0 && c) atomicAdd(&s_totR, c);
        __syncthreads();
        const uint32_t totR = s_totR;
        // pass 2: ranks of every L / R position; the t-th L position is swapped iff more than t R positions lie after it
        uint32_t runL = 0, runR = 0;
        for (uint32_t t0 = f + 1; t0 < l; t0 += kVgThreads) {
            const uint32_t i = t0 + tid;
            const bool valid = i < l;
            const uint32_t key = valid ? vkey(e[i]) : 0u;
            const bool isL = valid && key >= pk, isR = valid && key <= pk;
            const uint32_t bl = __ballot_sync(0xffffffffu, isL), br = __ballot_sync(0xffffffffu, isR);
            if (lane == 0) { s_wa[warp] = __popc(bl); s_wb[warp] = __popc(br); }
            __syncthreads();
            uint32_t pl = 0, pr = 0, tl = 0, tr = 0;
            for (int w = 0; w < kVgWarps; ++w) {
                if (w < warp) { pl += s_wa[w]; pr += s_wb[w]; }
                tl += s_wa[w]; tr += s_wb[w];
            }
            const uint32_t rankL = runL + pl + __popc(bl & lt_mask);
            const uint32_t rbefore = runR + pr + __popc(br & lt_mask);   // R positions before i
            if (isL) {
                posL[f + rankL] = i;
                const uint32_t rafter = totR - rbefore - (isR ? 1u : 0u);
                if (rafter > rankL) atomicMax(&s_m, rankL + 1);
            }
            if (isR) posR[f + (totR - 1 - rbefore)] = i;
            runL += tl; runR += tr;
            __syncthreads();
        }
        const uint32_t m = s_m, totL = runL;
        // pass 3: the m swaps touch distinct positions
        for (uint32_t t = tid; t < m; t += kVgThreads) vswap(e, posL[f + t], posR[f + t]);
        if (tid == 0) {
            uint32_t cut = m < totL ? posL[f + m] : UINT32_MAX;
            if (m > 0) cut = min(cut, posR[f + m - 1]);
            // children [cut, l) and [f, cut), both with the decremented depth
            const uint32_t cf[2] = {cut, f}, cl[2] = {l, cut};
            for (int h = 0; h < 2; ++h) {
                const uint32_t len = cl[h] - cf[h];
                if (len > kVgSmall) { s_f[s_sp] = cf[h]; s_l[s_sp] = cl[h]; s_d[s_sp] = d - 1; ++s_sp; }
                else if (len > 1) segs[s_nsmall++] = vg_seg(cf[h], len, d - 1);
            }
        }
        __syncthreads();
    }
    // ---- 3b. short segments, one thread each
    const uint32_t nsmall = s_nsmall;
    for (uint32_t s = tid; s < nsmall; s += kVgThreads) {
        const uint64_t g = segs[s];
        const uint32_t f = (uint32_t)(g >> 32), len = (uint32_t)(g >> 8) & 0xffffffu;
        vg_introsort_seq(e, f, f + len, (int)(g & 0xffu));
    }
    __syncthreads();
    // ---- 4. centroids: sequential f32 sums in sorted order, then / (float)count
    uint32_t run = 0;
    for (uint32_t t0 = 0; t0 < n; t0 += kVgThreads) {
        const uint32_t i = t0 + tid;
        const bool head = i < n && (i == 0 || vkey(e[i]) != vkey(e[i - 1]));
        const uint32_t bh = __ballot_sync(0xffffffffu, head);
        if (lane == 0) s_wa[warp] = __popc(bh);
        __syncthreads();
        uint32_t pre = 0, tot = 0;
        for (int w = 0; w < kVgWarps; ++w) { if (w < warp) pre += s_wa[w]; tot += s_wa[w]; }
        if (head) {
            const uint32_t key = vkey(e[i]);
            float sx = 0.0f, sy = 0.0f, sz = 0.0f, si = 0.0f;
            uint32_t j = i;
            for (; j < n && vkey(e[j]) == key; ++j) {
                const uint32_t p = (uint32_t)e[j];
                sx = x86_add(sx, X[p]); sy = x86_add(sy, Y[p]); sz = x86_add(sz, Z[p]); si = x86_add(si, I[p]);
            }
            const float cntf = __uint2float_rn(j - i);
            const int64_t q = o + run + pre + __popc(bh & lt_mask);
            A.sc.x()[q] = x86_div(sx, cntf); A.sc.y()[q] = x86_div(sy, cntf);
            A.sc.z()[q] = x86_div(sz, cntf); A.sc.i()[q] = x86_div(si, cntf);
        }
        run += tot;
        __syncthreads();
    }
    if (tid == 0) A.cnt[k] = run;
}

// out_off[0..K] = exclusive prefix of cnt, out_off[K+1] = number of overflow exits (one CTA)
__global__ void __launch_bounds__(1024) voxel_grid_offsets_kernel(const int64_t* __restrict__ cnt, const int32_t* __restrict__ status, int K,
                                                                  int64_t* __restrict__ out_off) {
    __shared__ int64_t s_w[32];
    __shared__ int64_t s_run;
    __shared__ unsigned s_ov;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_run = 0; s_ov = 0; }
    __syncthreads();
    for (int t0 = 0; t0 < K; t0 += 1024) {
        const int k = t0 + tid;
        const int64_t v = k < K ? cnt[k] : 0;
        if (k < K && status[k] == 1) atomicAdd(&s_ov, 1u);
        int64_t incl = v;
        for (int s = 1; s < 32; s <<= 1) { const int64_t u = __shfl_up_sync(0xffffffffu, incl, s); if (lane >= s) incl += u; }
        if (lane == 31) s_w[warp] = incl;
        __syncthreads();
        int64_t pre = 0, tot = 0;
        for (int w = 0; w < 32; ++w) { if (w < warp) pre += s_w[w]; tot += s_w[w]; }
        const int64_t run = s_run;
        if (k < K) out_off[k] = run + pre + incl - v;
        __syncthreads();
        if (tid == 0) s_run = run + tot;
        __syncthreads();
    }
    if (tid == 0) { out_off[K] = s_run; out_off[K + 1] = s_ov; }
}

// ordered compaction: centroids from the scratch, overflow-exit scans straight from the input (device-to-device)
__global__ void __launch_bounds__(256) voxel_grid_emit_kernel(PtrView src, const int64_t* __restrict__ off, DevCloud sc,
                                                              const int32_t* __restrict__ status, const int64_t* __restrict__ out_off, DevCloud out) {
    const int k = blockIdx.x;
    const int64_t m = out_off[k + 1] - out_off[k], si = off[k], di = out_off[k];
    const bool from_src = status[k] != 0;
    const float* x = from_src ? src.x : sc.x(); const float* y = from_src ? src.y : sc.y();
    const float* z = from_src ? src.z : sc.z(); const float* w = from_src ? src.i : sc.i();
    for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
        out.x()[di + i] = x[si + i]; out.y()[di + i] = y[si + i]; out.z()[di + i] = z[si + i]; out.i()[di + i] = w[si + i];
    }
}

// The filter over the K scans [off[k], off[k+1]) of `src`; make_out(out_off) allocates the output and returns it.
template <class MakeOut>
static int voxel_grid_run(ltr_ctx* ctx, const PtrView& src, const std::vector<int64_t>& off, const int64_t* d_off, float leaf,
                          int32_t* n_overflowed, MakeOut make_out) {
    if (!(leaf > 0.0f) || !std::isfinite(leaf)) return fail(ctx, LTR_ERR_INVALID, "voxel grid leaf size must be positive and finite (got %g)", (double)leaf);
    const int K = (int)off.size() - 1;
    int64_t max_chunk = 0;
    for (int k = 0; k < K; ++k) {
        const int64_t n = off[k + 1] - off[k];
        if (n >= ((int64_t)1 << 31)) return fail(ctx, LTR_ERR_UNSUPPORTED, "voxel grid: scan %d has %lld points (>= 2^31)", k, (long long)n);
        max_chunk = std::max(max_chunk, n);
    }
    max_chunk = std::max(max_chunk, std::min<int64_t>(off[K], env_points("LTR_VOXEL_GRID_CHUNK_POINTS", kVgChunkPoints, kVgChunkPoints)));
    void *p_ent = nullptr, *p_pos = nullptr, *p_segs = nullptr, *p_cnt = nullptr, *p_status = nullptr, *p_oo = nullptr;
    ScratchGuard g_ent(ctx, &p_ent), g_pos(ctx, &p_pos), g_segs(ctx, &p_segs), g_cnt(ctx, &p_cnt), g_status(ctx, &p_status), g_oo(ctx, &p_oo);
    CloudOwner g_sc;
    const size_t nk = (size_t)std::max(K, 1);
    LTR_TRY(dev_alloc(ctx, &p_cnt, nk * sizeof(int64_t)));
    LTR_TRY(dev_alloc(ctx, &p_status, nk * sizeof(int32_t)));
    LTR_TRY(dev_alloc(ctx, &p_oo, (size_t)(K + 2) * sizeof(int64_t)));
    if (off[K] > 0) {
        LTR_TRY(dev_alloc(ctx, &p_ent, (size_t)max_chunk * sizeof(uint64_t)));
        LTR_TRY(dev_alloc(ctx, &p_pos, (size_t)max_chunk * 2 * sizeof(uint32_t)));
        LTR_TRY(dev_alloc(ctx, &p_segs, (size_t)max_chunk * sizeof(uint64_t)));
        LTR_TRY(cloud_new(ctx, off[K], &g_sc));
    }
    const DevCloud sc = g_sc.get() >= 0 ? ctx->clouds[g_sc.get()] : DevCloud();
    for (int k0 = 0; k0 < K;) {
        int k1 = k0 + 1;
        while (k1 < K && off[k1 + 1] - off[k0] <= max_chunk) ++k1;
        VgArgs a;
        a.src = src; a.off = d_off; a.k0 = k0; a.base = off[k0]; a.leaf = leaf;
        a.ent = (uint64_t*)p_ent; a.posL = (uint32_t*)p_pos; a.posR = (uint32_t*)p_pos + max_chunk; a.segs = (uint64_t*)p_segs;
        a.sc = sc; a.cnt = (int64_t*)p_cnt; a.status = (int32_t*)p_status;
        voxel_grid_kernel<<<k1 - k0, kVgThreads, 0, ctx->stream>>>(a);
        LTR_LAUNCH_CHECK(ctx);
        k0 = k1;
    }
    if (K > 0) {
        voxel_grid_offsets_kernel<<<1, 1024, 0, ctx->stream>>>((const int64_t*)p_cnt, (const int32_t*)p_status, K, (int64_t*)p_oo);
        LTR_LAUNCH_CHECK(ctx);
    }
    std::vector<int64_t> oo((size_t)K + 2, 0);
    if (K > 0) {
        LTR_CUDA(ctx, cudaMemcpyAsync(oo.data(), p_oo, (size_t)(K + 2) * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        LTR_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    if (n_overflowed) *n_overflowed = (int32_t)oo[(size_t)K + 1];
    oo.resize((size_t)K + 1);
    DevCloud out;
    LTR_TRY(make_out(oo, &out));
    if (K > 0 && oo[(size_t)K] > 0) {
        voxel_grid_emit_kernel<<<K, 256, 0, ctx->stream>>>(src, d_off, sc, (const int32_t*)p_status, (const int64_t*)p_oo, out);
        LTR_LAUNCH_CHECK(ctx);
    }
    return LTR_OK;
}

}  // namespace ltr

using namespace ltr;

extern "C" {

int ltr_voxel_grid(ltr_ctx* ctx, ltr_cloud in, float leaf, ltr_cloud* out, int32_t* overflowed) {
    ApiTrace tr__(ctx, "ltr_voxel_grid");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevCloud* c;
    LTR_TRY(cloud_get(ctx, in, &c));
    const DevCloud src = *c;
    const std::vector<int64_t> off = {0, src.n};
    void* p_off = nullptr;
    ScratchGuard g_off(ctx, &p_off);
    LTR_TRY(dev_alloc(ctx, &p_off, 2 * sizeof(int64_t)));
    LTR_CUDA(ctx, cudaMemcpyAsync(p_off, off.data(), 2 * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
    int32_t nov = 0;
    CloudOwner h;
    LTR_TRY(voxel_grid_run(ctx, view(src), off, (const int64_t*)p_off, leaf, &nov, [&](const std::vector<int64_t>& oo, DevCloud* o) {
        LTR_TRY(cloud_new(ctx, oo[1], &h));
        *o = ctx->clouds[h.get()];
        return (int)LTR_OK;
    }));
    *out = h.release();
    if (overflowed) *overflowed = nov;
    return LTR_OK;
}

int ltr_voxel_grid_per_keyframe(ltr_ctx* ctx, ltr_scanset in, float leaf, ltr_scanset* out, int32_t* n_overflowed) {
    ApiTrace tr__(ctx, "ltr_voxel_grid_per_keyframe");
    if (!ctx || !out) return fail(ctx, LTR_ERR_INVALID, "null argument");
    DevScanSet* s;
    LTR_TRY(scanset_get(ctx, in, &s));
    const DevScanSet ss = *s;   // copy: scanset_new may reallocate the handle table
    ScanSetOwner h;
    LTR_TRY(voxel_grid_run(ctx, view(ss.pts), ss.h_off, ss.d_off, leaf, n_overflowed, [&](const std::vector<int64_t>& oo, DevCloud* o) {
        LTR_TRY(scanset_new(ctx, oo, &h));
        *o = ctx->scansets[h.get()].pts;
        return (int)LTR_OK;
    }));
    *out = h.release();
    return LTR_OK;
}

}  // extern "C"
