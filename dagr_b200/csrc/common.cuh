// common.cuh -- shared helpers for libdagr_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/dagr_b200.h"

#ifndef __CUDA_ARCH__
#define DAGR_HOST 1
#endif

void dagr_set_error(const char *fmt, ...);

#define DAGR_CHECK_ARG(cond, msg)                                              \
    do { if (!(cond)) { dagr_set_error("%s: %s", __func__, msg); return DAGR_E_ARG; } } while (0)

#define DAGR_CHECK_LAUNCH()                                                    \
    do { cudaError_t e__ = cudaGetLastError();                                 \
         if (e__ != cudaSuccess) { dagr_set_error("%s: %s", __func__, cudaGetErrorString(e__)); \
                                   return DAGR_E_CUDA; } } while (0)

#define DAGR_CUDA(call)                                                        \
    do { cudaError_t e__ = (call);                                             \
         if (e__ != cudaSuccess) { dagr_set_error("%s: %s", __func__, cudaGetErrorString(e__)); \
                                   return DAGR_E_CUDA; } } while (0)

// Opt-in dynamic shared memory of a kernel, RAISE-ONLY.  The attribute is process-global state of the function: a launcher that
// sets it to "this launch's size" lowers it again for the next, smaller launch.  A captured kernel node keeps the value it was
// captured with, but tools that re-launch the nodes of a graph one by one (ncu's default per-node graph profiling) use the
// CURRENT value and a node that needs more fails to launch.  capi.cu keeps the per-function maximum (and saves the driver
// call on every later launch).
cudaError_t dagr_allow_smem_impl(const void *kernel, size_t bytes, bool max_carveout);
template <class K> static inline cudaError_t dagr_allow_smem(K kernel, size_t bytes, bool max_carveout = false)
{
    return dagr_allow_smem_impl(reinterpret_cast<const void *>(kernel), bytes, max_carveout);
}

static inline int dagr_div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// Plane mode of the image kernels (several hybrid cameras as the samples of one step): the image is a plane array
// [n][C][h][w] and sample b reads plane plane[b * stride] alone, sampled as a batch of one (b = 0, Bi = 1: the depth
// coordinate is exactly 0), i.e. with the bits of that sample in a B = 1 forward.  The plane table is device data that the
// launch cannot check, so a value outside [0, n) is clamped (it selects a wrong plane, never memory outside the array).
struct ImgPlanes {
    const int32_t *plane;
    int stride, n;
};
__device__ __forceinline__ int img_plane(const ImgPlanes &pl, int b)
{
    return min(max(__ldg(pl.plane + (int64_t)b * pl.stride), 0), pl.n - 1);
}

// exclusive prefix sum of n ints (graph.cu); blocksums: int[dagr_scan_blocks(n) + 2]; the grand total is left in
// blocksums[dagr_scan_blocks(n)]
int scan_exclusive(const int *in, int *out, int64_t n, int *blocksums, cudaStream_t st);

// xa rows are stored half-major [2][N][8]; inside each 32-byte half-row the two 16-byte chunks are swapped when bit 2 of
// the row index is set.  A staged copy of the rows (TMA keeps them contiguous) then spreads a warp's random row gathers
// over all eight 16-byte bank groups instead of four (LDS.128 conflict degree ~3.4 -> ~2.3).
#define XA_SWZ(p) ((int)(((p) >> 2) & 1))

// order-preserving float <-> uint32 encoding (0 is below every encoded value -> "empty")
__device__ __forceinline__ uint32_t enc_ordered(float f)
{
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float dec_ordered(uint32_t e)
{
    uint32_t u = (e & 0x80000000u) ? (e & 0x7fffffffu) : ~e;
    return __uint_as_float(u);
}

// fp32 FMA on both halves of a float2: d = a*b + c, round-to-nearest on each.  Hopper has no packed fp32 FMA, so this is
// two FFMA; the kernels keep their paired accumulator layout.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// degree-1 open B-spline basis in 2-D (torch_spline_conv semantics): 4 (weight, slot) pairs
// for pseudo coordinates (ax, ay); kernel_size ks per dim.
__device__ __forceinline__ void spline_basis2(float ax, float ay, int ks, float w[4], int slot[4])
{
    float vx = ax * (float)(ks - 1), vy = ay * (float)(ks - 1);
    float fx = vx - floorf(vx), fy = vy - floorf(vy);
    int ix = (int)vx, iy = (int)vy;                 // C-cast truncation like the reference
#pragma unroll
    for (int s = 0; s < 4; s++) {
        int kx = s & 1, ky = (s >> 1) & 1;
        int sx = (ix + kx) % ks, sy = (iy + ky) % ks;
        if (sx < 0) sx += ks;
        if (sy < 0) sy += ks;
        slot[s] = sx + ks * sy;
        // basis *= k ? frac : 1-frac, x first then y (same association as the reference loop)
        w[s] = (kx ? fx : 1.f - fx) * (ky ? fy : 1.f - fy);
    }
}
