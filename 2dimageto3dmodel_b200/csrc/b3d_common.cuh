// Shared helpers of libb3d (sm_90a).  Error plumbing for the C ABI, launch accounting,
// NaN-propagating clamps (torch.clamp semantics) and warp/block reductions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b3d.h"

namespace b3d {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
// kernel-variant record of the calling thread's most recent convolution entry point (b3d_last_variant)
void clear_variant();
void add_variant(const char* fmt, ...);

#define B3D_REQUIRE(cond, code, ...)      \
    do {                                  \
        if (!(cond)) {                    \
            b3d::set_error(__VA_ARGS__);  \
            return (code);                \
        }                                 \
    } while (0)

#define B3D_CHECK_ALIGNED(p)                                                                   \
    B3D_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15u) == 0, B3D_EALIGN, "%s: %s not 16-byte aligned", \
                __func__, #p)

#define B3D_CUDA_OK(expr)                                                                      \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            b3d::set_error("%s: %s failed: %s", __func__, #expr, cudaGetErrorString(e__));     \
            return B3D_ECUDA;                                                                  \
        }                                                                                      \
    } while (0)

#define B3D_LAUNCH_OK()                                                                        \
    do {                                                                                       \
        cudaError_t e__ = cudaGetLastError();                                                  \
        if (e__ != cudaSuccess) {                                                              \
            b3d::set_error("%s: kernel launch failed: %s", __func__, cudaGetErrorString(e__)); \
            return B3D_ECUDA;                                                                  \
        }                                                                                      \
        b3d::count_launch();                                                                   \
    } while (0)

// torch.clamp propagates NaN; fminf/fmaxf do not.
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) {
    return x < lo ? lo : (x > hi ? hi : x);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum over the block; result valid in thread 0.  `red` is >= 32 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (w == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        v = lane < nw ? red[lane] : 0.f;
        v = warp_sum(v);
    }
    return v;
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// dpg[b, original index] = d/d(grid coords) of every bin-sorted point, gathered at its 8 corners of dgrid [B,V,V,V]
// (csrc/vox_kernels.cu; b3d_vox_gather masks dgrid first, the mode-P silhouette backward has masked it already)
int vox_gather_launch(const float* sorted, const int32_t* bin_start, const float* dgrid, int B, int N, int V, int mode,
                      float* dpg, cudaStream_t st);

}  // namespace b3d
