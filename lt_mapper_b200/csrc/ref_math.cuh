// Device restatement of the scalar arithmetic of the LT-removert hot path, bit-exact with the reference's
// x86-64 Release build (no FMA contraction, IEEE float/double, glibc atan2f):
//   cart2sph            ltremovert/src/utility.cpp:38-51
//   rad2deg             ltremovert/src/utility.cpp:53-56
//   pixel index         ltremovert/src/utility.cpp:118-123 == ltremovert/src/Removerter.cpp:133-138
//   transformPointCloud PCL semantics at ltremovert/src/utility.cpp:70-71, 164-165, 198-199
// Every operation is spelled with round-to-nearest intrinsics so the compiler cannot contract a
// multiply-add into an FMA regardless of -fmad; glibc's atan2f (<= 2.39) is Sun's fdlibm algorithm
// (public domain e_atan2f.c / s_atanf.c), written out here in IEEE float ops.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ltr {

#define LTR_DEV __device__ __forceinline__

LTR_DEV float fm(float a, float b) { return __fmul_rn(a, b); }
LTR_DEV float fa(float a, float b) { return __fadd_rn(a, b); }
LTR_DEV float fs(float a, float b) { return __fsub_rn(a, b); }
LTR_DEV float fd(float a, float b) { return __fdiv_rn(a, b); }
LTR_DEV double dm(double a, double b) { return __dmul_rn(a, b); }
LTR_DEV double da(double a, double b) { return __dadd_rn(a, b); }

LTR_DEV float ref_atanf(float x) {
    const int32_t hx = __float_as_int(x);
    const int32_t ix = hx & 0x7fffffff;
    float hi, lo;
    int id;
    if (ix >= 0x4c000000) {  // |x| >= 2^25 (glibc 2.39 s_atanf.c; the oracle's copy is checked against the container's libm around this value)
        if (ix > 0x7f800000) return fa(x, x);
        const float r = fa(1.5707962513e+00f, 7.5497894159e-08f);
        return (hx > 0) ? r : -r;
    }
    if (ix < 0x3ee00000) {  // |x| < 0.4375
        if (ix < 0x31000000) return x;
        id = -1; hi = 0.0f; lo = 0.0f;
    } else {
        x = fabsf(x);
        if (ix < 0x3f980000) {
            if (ix < 0x3f300000) { id = 0; hi = 4.6364760399e-01f; lo = 5.0121582440e-09f; x = fd(fs(fm(2.0f, x), 1.0f), fa(2.0f, x)); }
            else                 { id = 1; hi = 7.8539812565e-01f; lo = 3.7748947079e-08f; x = fd(fs(x, 1.0f), fa(x, 1.0f)); }
        } else {
            if (ix < 0x401c0000) { id = 2; hi = 9.8279368877e-01f; lo = 3.4473217170e-08f; x = fd(fs(x, 1.5f), fa(1.0f, fm(1.5f, x))); }
            else                 { id = 3; hi = 1.5707962513e+00f; lo = 7.5497894159e-08f; x = fd(-1.0f, x); }
        }
    }
    const float z = fm(x, x);
    const float w = fm(z, z);
    const float s1 = fm(z, fa(3.3333334327e-01f, fm(w, fa(1.4285714924e-01f, fm(w, fa(9.0908870101e-02f,
                     fm(w, fa(6.6610731184e-02f, fm(w, fa(4.9768779427e-02f, fm(w, 1.6285819933e-02f)))))))))));
    const float s2 = fm(w, fa(-2.0000000298e-01f, fm(w, fa(-1.1111110449e-01f, fm(w, fa(-7.6918758452e-02f,
                     fm(w, fa(-5.8335702866e-02f, fm(w, -3.6531571299e-02f)))))))));
    if (id < 0) return fs(x, fm(x, fa(s1, s2)));
    const float r = fs(hi, fs(fs(fm(x, fa(s1, s2)), lo), x));
    return (hx < 0) ? -r : r;
}

LTR_DEV float ref_atan2f(float y, float x) {
    const float tiny = 1.0e-30f;
    const float pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f, pi_lo = -8.7422776573e-08f;
    const int32_t hx = __float_as_int(x), hy = __float_as_int(y);
    const int32_t ix = hx & 0x7fffffff, iy = hy & 0x7fffffff;
    if (ix > 0x7f800000 || iy > 0x7f800000) return fa(x, y);
    if (hx == 0x3f800000) return ref_atanf(y);
    const int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
    if (iy == 0) {
        if (m < 2) return y;
        return (m == 2) ? fa(pi, tiny) : fs(-pi, tiny);
    }
    if (ix == 0) return (hy < 0) ? fs(-pi_o_2, tiny) : fa(pi_o_2, tiny);
    if (ix == 0x7f800000) {
        if (iy == 0x7f800000) {
            switch (m) {
                case 0: return fa(pi_o_4, tiny);
                case 1: return fs(-pi_o_4, tiny);
                case 2: return fa(fm(3.0f, pi_o_4), tiny);
                default: return fs(fm(-3.0f, pi_o_4), tiny);
            }
        } else {
            switch (m) {
                case 0: return 0.0f;
                case 1: return -0.0f;
                case 2: return fa(pi, tiny);
                default: return fs(-pi, tiny);
            }
        }
    }
    if (iy == 0x7f800000) return (hy < 0) ? fs(-pi_o_2, tiny) : fa(pi_o_2, tiny);
    const int32_t k = (iy - ix) >> 23;
    float z;
    if (k > 60) z = fa(pi_o_2, fm(0.5f, pi_lo));
    else if (hx < 0 && k < -60) z = 0.0f;
    else z = ref_atanf(fabsf(fd(y, x)));
    switch (m) {
        case 0: return z;
        case 1: return __int_as_float(__float_as_int(z) ^ 0x80000000);
        case 2: return fs(pi, fs(z, pi_lo));
        default: return fs(fs(z, pi_lo), pi);
    }
}

struct Sph { float az, el, r; };

// cart2sph (utility.cpp:38-51)
LTR_DEV Sph cart2sph(float x, float y, float z) {
    Sph s;
    const float xx = fm(x, x), yy = fm(y, y);
    const float rho2 = fa(xx, yy);
    s.az = ref_atan2f(y, x);
    s.el = ref_atan2f(z, __fsqrt_rn(rho2));
    s.r = __fsqrt_rn(fa(rho2, fm(z, z)));
    return s;
}

// rad2deg (utility.cpp:53-56): (float)((double)rad * 180.0 / M_PI)
LTR_DEV float rad2deg(float r) {
    return __double2float_rn(__ddiv_rn(dm((double)r, 180.0), 3.14159265358979323846));
}

// std::round(float): halfway cases away from zero, exact
LTR_DEV float round_half_away(float v) {
    const float t = truncf(v);
    const float f = fs(v, t);  // exact
    if (f >= 0.5f) return fa(t, 1.0f);
    if (f <= -0.5f) return fs(t, 1.0f);
    return t;
}

struct ImgShape { int rows, cols; float vfov, hfov; };

// pixel index (utility.cpp:118-123)
LTR_DEV void pixel_index(const Sph& s, const ImgShape& g, int* row, int* col) {
    const float rr = round_half_away(fm((float)g.rows, fs(1.0f, fd(fa(rad2deg(s.el), fd(g.vfov, 2.0f)), fs(g.vfov, 0.0f)))));
    const float cc = round_half_away(fm((float)g.cols, fd(fa(rad2deg(s.az), fd(g.hfov, 2.0f)), fs(g.hfov, 0.0f))));
    *row = (int)fminf(fmaxf(rr, 0.0f), (float)(g.rows - 1));
    *col = (int)fminf(fmaxf(cc, 0.0f), (float)(g.cols - 1));
}

// pcl::transformPointCloud, one point, 3x4 row-major double matrix m (see include/ltr_b200.h transform_order)
LTR_DEV void transform_point(const double* __restrict__ m, int order, float x, float y, float z, float* ox, float* oy, float* oz) {
    const double px = (double)x, py = (double)y, pz = (double)z;
    if (order == 0) {
        *ox = __double2float_rn(da(da(da(dm(m[0], px), dm(m[1], py)), dm(m[2], pz)), m[3]));
        *oy = __double2float_rn(da(da(da(dm(m[4], px), dm(m[5], py)), dm(m[6], pz)), m[7]));
        *oz = __double2float_rn(da(da(da(dm(m[8], px), dm(m[9], py)), dm(m[10], pz)), m[11]));
    } else {
        *ox = __double2float_rn(da(da(da(m[3], dm(px, m[0])), dm(py, m[1])), dm(pz, m[2])));
        *oy = __double2float_rn(da(da(da(m[7], dm(px, m[4])), dm(py, m[5])), dm(pz, m[6])));
        *oz = __double2float_rn(da(da(da(m[11], dm(px, m[8])), dm(py, m[9])), dm(pz, m[10])));
    }
}

// transformGlobalMapToLocal for one map point (utility.cpp:70-71): the keyframe's inverse pose, then the extrinsic unless it is exactly
// the identity (ext: base2lidar rows 0..2)
LTR_DEV void map_to_sensor(const double* __restrict__ inv_pose, const double* __restrict__ ext, int ext_identity, int order, float x, float y,
                           float z, float* lx, float* ly, float* lz) {
    transform_point(inv_pose, order, x, y, z, lx, ly, lz);
    if (!ext_identity) transform_point(ext, order, *lx, *ly, *lz, lx, ly, lz);
}

// local2global of a scan point (utility.cpp:164-165): the extrinsic `ext` (3x4 rows), skipped when null because it is exactly the identity,
// then the pose (rows 0..2).  The reference passes different extrinsics on different paths (DESIGN.md §5.1): base2lidar (ltr_ctx::d_ext)
// for the kNN diff (Session.cpp:545) and ICP, lidar2base (d_ext + 12) for scan-side removal and mergeScansWithinGlobalCoordUtil.  The
// paths that move points back all use map_to_sensor with base2lidar (Session.cpp:603-604, utility.cpp:198-199).
LTR_DEV void scan_to_global(const double* __restrict__ pose, const double* __restrict__ ext, int order, float* x, float* y, float* z) {
    if (ext) transform_point(ext, order, *x, *y, *z, x, y, z);
    transform_point(pose, order, *x, *y, *z, x, y, z);
}

// ((m0 x + m1 y) + m2 z) + m3 in f32, m = one row of a row-major float 4x4 (PCL's Matrix4f applied to a point)
LTR_DEV float frow(const float* m, float x, float y, float z) { return fa(fa(fa(fm(m[0], x), fm(m[1], y)), fm(m[2], z)), m[3]); }

// The registration of ltr_knn_diff_refined and ltr_scanside_split_refined (Session.cpp:565): a global point of keyframe kf moved by the
// float 4x4 T16 + 16 kf with frow when accept[kf] != 0.  T16 == null: no refinement, the point stays.
LTR_DEV void refine_point(const float* __restrict__ T16, const uint8_t* __restrict__ accept, int kf, float* x, float* y, float* z) {
    if (!T16 || !accept[kf]) return;
    const float* m = T16 + 16 * (size_t)kf;
    const float nx = frow(m, *x, *y, *z), ny = frow(m + 4, *x, *y, *z), nz = frow(m + 8, *x, *y, *z);
    *x = nx; *y = ny; *z = nz;
}

// FLANN L2_Simple<float> squared distance: ((dx*dx) + dy*dy) + dz*dz with dx = query - point
LTR_DEV float l2_simple(float qx, float qy, float qz, float px, float py, float pz) {
    const float dx = fs(qx, px), dy = fs(qy, py), dz = fs(qz, pz);
    return fa(fa(fm(dx, dx), fm(dy, dy)), fm(dz, dz));
}

// The KT smallest values pushed so far in ascending order (+inf where fewer were pushed); seen counts the pushes.  Every search pushes the
// points of one grid, whose point indices are 32-bit, so seen cannot wrap.
template <int KT>
struct TopK {
    float d[KT];
    uint32_t seen;
    LTR_DEV void init() {
#pragma unroll
        for (int j = 0; j < KT; ++j) d[j] = __int_as_float(0x7f800000);
        seen = 0;
    }
    // true when v entered the list
    LTR_DEV bool push(float v) {
        ++seen;
        if (!(v < d[KT - 1])) return false;
        d[KT - 1] = v;
#pragma unroll
        for (int j = KT - 1; j > 0; --j)
            if (d[j] < d[j - 1]) { const float t = d[j]; d[j] = d[j - 1]; d[j - 1] = t; }
        return true;
    }
    LTR_DEV bool has(int k) const { return seen >= (uint32_t)k; }
    // The reference's mean of the k nearest squared distances: accumulate(..., 0.0) in double over the min(seen, k) smallest, ascending,
    // then float(sum) / float(k) (Session.cpp:470-471, 592-594; Removerter.cpp:1052-1053, 1097-1098).
    LTR_DEV float mean(int k) const {
        const int cnt = has(k) ? k : (int)seen;
        double sum = 0.0;
#pragma unroll
        for (int j = 0; j < KT; ++j) if (j < cnt) sum = da(sum, (double)d[j]);
        return fd(__double2float_rn(sum), (float)k);
    }
    // the kNN diff's test |mean| < thr: "near"
    LTR_DEV bool near(int k, float thr) const { return fabsf(mean(k)) < thr; }
};

// The thresholded kNN decision, 1 = far and 0 = near, of the query q over the 27 cells around its cell (cx, cy, cz) in a grid of dim
// cells, KT >= k.  rows(y, z, xa, xb, &s, &e) gives the points pts[s, e) of the cells [xa, xb] of row (y, z).  The caller's cells are wide
// enough that a true k-th neighbour outside the block already makes the mean >= thr (knn.cu and delta.cu prove it for their grids), so
// fewer than k points in the block mean "far".
template <int KT, class Rows>
LTR_DEV uint8_t knn_label_27(Rows rows, const float4* __restrict__ pts, int cx, int cy, int cz, const int (&dim)[3], float qx, float qy,
                             float qz, int k, float thr) {
    TopK<KT> b;
    b.init();
    const int x0 = max(cx - 1, 0), x1 = min(cx + 1, dim[0] - 1);
    if (x0 <= x1) {
        // rows of 3 x-adjacent cells, the query's own row first: most points have their k neighbours right there and leave through the
        // early exit below
        // (dy, dz) + 1 packed 2 bits per step: dy = {0,-1,1,0,0,-1,1,-1,1}, dz = {0,0,0,-1,1,-1,-1,1,1}
        const unsigned pack_dy = 0x22161U, pack_dz = 0x28215U;
#pragma unroll 1
        for (int o = 0; o < 9; ++o) {
            const int z = cz + (int)((pack_dz >> (2 * o)) & 3u) - 1, y = cy + (int)((pack_dy >> (2 * o)) & 3u) - 1;
            if (z < 0 || z >= dim[2] || y < 0 || y >= dim[1]) continue;
            uint32_t s, e;
            rows(y, z, x0, x1, &s, &e);
            for (uint32_t p = s; p < e; ++p) {
                const float4 t = pts[p];
                // Early exit: the final k smallest distances are element-wise <= the current ones, and the double sum, its float
                // rounding and the division are monotone, so "current mean < thr" already decides "near".  Short lists check after
                // each insertion, long ones after each row.
                if (b.push(l2_simple(qx, qy, qz, t.x, t.y, t.z)) && KT <= 4 && b.has(k) && b.near(k, thr)) return 0;
            }
            if (KT > 4 && b.has(k) && b.near(k, thr)) return 0;
        }
    }
    return (b.has(k) && b.near(k, thr)) ? 0 : 1;
}

// A target of n < k points, pt(p) for p < n: PCL's nearestKSearch returns all n of them (ascending) and the reference still divides
// their sum by k (Session.cpp:470-471, 592-594).  Brute force.
template <int KT, class Pt>
LTR_DEV uint8_t knn_label_all(int n, Pt pt, float qx, float qy, float qz, int k, float thr) {
    TopK<KT> b;
    b.init();
    for (int p = 0; p < n; ++p) {
        const float4 t = pt(p);
        b.push(l2_simple(qx, qy, qz, t.x, t.y, t.z));
    }
    return b.near(k, thr) ? 0 : 1;
}

}  // namespace ltr
