// Small device helpers shared by the kernels of util.cu and project.cu.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ltr {

// keyframe of element i in a segment list: off[lo] <= i < off[lo + 1] for the K segments off[0..K]
__device__ __forceinline__ int find_kf(const int64_t* __restrict__ off, int K, int64_t i) {
    int lo = 0, hi = K;  // off[lo] <= i < off[hi]
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (off[mid] <= i) lo = mid; else hi = mid; }
    return lo;
}

// ------------------------------------------------------------------------------------------------
// block-wide rank of a predicate (stable): returns the number of lower-indexed threads with pred set
// and the block total.  blockDim.x must be a multiple of 32 and <= 1024.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int block_rank(bool pred, int* total, int* s_warp /* 33 ints */) {
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    const unsigned b = __ballot_sync(0xffffffffu, pred);
    const int wrank = __popc(b & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    if (warp == 0) {
        int v = lane < nwarp ? s_warp[lane] : 0;
        int incl = v;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += t; }
        s_warp[lane] = incl - v;
        if (lane == 31) s_warp[32] = incl;
    }
    __syncthreads();
    const int r = s_warp[warp] + wrank;
    *total = s_warp[32];
    __syncthreads();
    return r;
}

}  // namespace ltr
