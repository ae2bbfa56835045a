// common.cuh -- shared helpers for libdagr_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/dagr_b200.h"

#ifndef __CUDA_ARCH__
#define DAGR_HOST 1
#endif

void dagr_set_error(const char *fmt, ...);

// The _AS forms name `who` in the error instead of the enclosing function: a launcher shared by several entry points passes
// the entry point's __func__, so dagr_last_error() names the function the caller called.
#define DAGR_CHECK_ARG_AS(who, cond, msg)                                      \
    do { if (!(cond)) { dagr_set_error("%s: %s", who, msg); return DAGR_E_ARG; } } while (0)
#define DAGR_CHECK_ARG(cond, msg) DAGR_CHECK_ARG_AS(__func__, cond, msg)

#define DAGR_CHECK_LAUNCH_AS(who)                                              \
    do { cudaError_t e__ = cudaGetLastError();                                 \
         if (e__ != cudaSuccess) { dagr_set_error("%s: %s", who, cudaGetErrorString(e__)); \
                                   return DAGR_E_CUDA; } } while (0)
#define DAGR_CHECK_LAUNCH() DAGR_CHECK_LAUNCH_AS(__func__)

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

// Map formats of the image-sampling kernels (their map element type MT): fp32 maps are NCHW [B][C][h][w] (the TF32 image
// branch), bf16 maps are NHWC [B][h][w][C] (the bf16 image branch's channels_last taps).  map_ld / map_ldg (read-only path)
// return element (z, c, y, x) of either as fp32; bf16 -> fp32 is exact, so a bf16 map samples to the bits of its fp32 upcast.
__device__ __forceinline__ float map_ld(const float *__restrict__ m, int C, int h, int w, int z, int c, int y, int x)
{
    return m[(((int64_t)z * C + c) * h + y) * w + x];
}
__device__ __forceinline__ float map_ld(const __nv_bfloat16 *__restrict__ m, int C, int h, int w, int z, int c, int y, int x)
{
    return __bfloat162float(m[(((int64_t)z * h + y) * w + x) * C + c]);
}
__device__ __forceinline__ float map_ldg(const float *__restrict__ m, int C, int h, int w, int z, int c, int y, int x)
{
    return __ldg(m + (((int64_t)z * C + c) * h + y) * w + x);
}
__device__ __forceinline__ float map_ldg(const __nv_bfloat16 *__restrict__ m, int C, int h, int w, int z, int c, int y, int x)
{
    return __bfloat162float(__ldg(m + (((int64_t)z * h + y) * w + x) * C + c));
}

// grid_sample(align_corners=True) of one (x, y, batch) position: weights and corner offsets, mirroring
// _sample_features (net.py:207-221): normalise with the event resolution, unnormalise with the map size.
struct Bilin {
    int x0, y0, z0;
    float tx, ty, tz;
};
__device__ __forceinline__ Bilin bilin_setup(float posx, float posy, int b, float width, float height, int Bi, int h, int w)
{
    const float gx = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fmul_rn(posx, width)), width - 1.f), 1.f);
    const float gy = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fmul_rn(posy, height)), height - 1.f), 1.f);
    const float bs = (float)(Bi > 1 ? Bi : 2);
    const float gz = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, (float)b), bs - 1.f), 1.f);
    const float ix = __fmul_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), (float)(w - 1));
    const float iy = __fmul_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), (float)(h - 1));
    const float iz = __fmul_rn(__fmul_rn(__fadd_rn(gz, 1.f), 0.5f), (float)(Bi - 1));
    Bilin r;
    const float x0f = floorf(ix), y0f = floorf(iy), z0f = floorf(iz);
    r.x0 = (int)x0f; r.y0 = (int)y0f; r.z0 = (int)z0f;
    r.tx = ix - x0f; r.ty = iy - y0f; r.tz = iz - z0f;
    return r;
}
// One in-bounds corner of a trilinear sample: map element (z, y, x) and its weight's factors.  w() is the weight in the
// oracle's association; each kernel calls it where its arithmetic has always had it (after the load in the per-channel loops,
// before the loads in the voxel kernel's 8-channel path), so the shared loop leaves every kernel's instruction order as it was.
struct BilinTap {
    int z, y, x;
    float wx, wy, wz;
    __device__ __forceinline__ float w() const { return wx * wy * wz; }
};
// The trilinear taps of q in a [Bi][h][w] map with zero padding: f(tap) for each in-bounds corner, in the order dz, dy, dx.
// Every image-sampling kernel walks its taps here and accumulates acc += v * tap.w(), so all of them (and the oracle) share
// one tap order and one fp32 arithmetic; only the loader of v differs.
template <typename F>
__device__ __forceinline__ void bilin_taps(const Bilin &q, int Bi, int h, int w, F &&f)
{
#pragma unroll
    for (int dz = 0; dz < 2; dz++) {
        const int z = q.z0 + dz;
        const float wz = dz ? q.tz : 1.f - q.tz;
        if (z < 0 || z >= Bi) continue;
#pragma unroll
        for (int dy = 0; dy < 2; dy++) {
            const int y = q.y0 + dy;
            const float wy = dy ? q.ty : 1.f - q.ty;
            if (y < 0 || y >= h) continue;
#pragma unroll
            for (int dx = 0; dx < 2; dx++) {
                const int x = q.x0 + dx;
                const float wx = dx ? q.tx : 1.f - q.tx;
                if (x < 0 || x >= w) continue;
                f(BilinTap{z, y, x, wx, wy, wz});
            }
        }
    }
}

// exclusive prefix sum of n ints (graph.cu); blocksums: int[dagr_scan_blocks(n) + 2]; the grand total is left in
// blocksums[dagr_scan_blocks(n)]
int scan_exclusive(const int *in, int *out, int64_t n, int *blocksums, cudaStream_t st);

// exclusive prefix sum of one int per thread over the CTA (every thread must call it); *total = the CTA's sum.
// smem: int[32] of the caller's shared memory.
__device__ __forceinline__ int block_exclusive_scan(int v, int *total, int *smem /*[32]*/)
{
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) smem[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int w = (lane < (blockDim.x >> 5)) ? smem[lane] : 0;
        int wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            int o = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += o;
        }
        smem[lane] = wi - w;            // exclusive warp offsets
        if (lane == 31) *total = wi;
    }
    __syncthreads();
    int res = smem[wid] + incl - v;
    __syncthreads();
    return res;
}

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

// torch.div(a, b, rounding_mode='floor') for fp32 (c10::div_floor_floating), needed because
// floorf(a/b) differs when the rounded quotient lands on an integer from below.
__device__ __forceinline__ float div_floor_f32(float a, float b)
{
    const float mod = fmodf(a, b);
    float div = __fdiv_rn(__fsub_rn(a, mod), b);
    if ((mod != 0.f) && ((b < 0.f) != (mod < 0.f))) div -= 1.f;
    float fl;
    if (div != 0.f) {
        fl = floorf(div);
        if (div - fl > 0.5f) fl += 1.f;
    } else {
        fl = copysignf(0.f, __fdiv_rn(a, b));
    }
    return fl;
}

// pixel position of a pooled voxel (pool1 in conv_l1.cu, pool2..4 in coarse.cu)
__device__ __forceinline__ int round_to_pixel(float mean, int size)
{
    // floor((pos + 1e-5) / (1/size))   (pooling.py:47-49), wh_inv = fl(1/size)
    const float inv = __frcp_rn((float)size);
    const float q = div_floor_f32(__fadd_rn(mean, 1e-5f), inv);
    const int k = (int)q;
    return min(max(k, 0), size - 1);
}

// fp32 FMA on both halves of a float2: d = a*b + c, round-to-nearest on each.  Hopper has no packed fp32 FMA, so this is
// two FFMA; the kernels keep their paired accumulator layout.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// ---- 3xTF32 on tensor cores (mma.sync.m16n8k8, used by the per-voxel conv kernels of conv_l1.cu and build_l1.cu) ----------
// x = hi + lo with hi = cvt.rna.tf32(x) and lo = x - hi (exact); a product is summed as a_lo*b_hi + a_hi*b_lo + a_hi*b_hi,
// relative error ~1e-6 against the fp32 sum.  Fragment order of m16n8k8 (g = lane >> 2, t = lane & 3):
//   A (row-major 16 x 8): a0 = A[g][t], a1 = A[g+8][t], a2 = A[g][t+4], a3 = A[g+8][t+4]
//   B (col-major 8 x 8):  b0 = B[t][g], b1 = B[t+4][g]
//   C (16 x 8):           c01 = (C[g][2t], C[g][2t+1]), c23 = (C[g+8][2t], C[g+8][2t+1])
// The weight fragments come split on the host, one float4 per lane and n-tile: (hi b0, hi b1, lo b0, lo b1).
// hi is rounded with integer ops: sm_90 has no instruction for cvt.rna.tf32.f32, and ptxas expands it to a non-finite test,
// an add, a select and a mask per value.  (x + 0x1000) & 0xffffe000 is that expansion without the test: the same bits for
// every finite x (round to nearest, ties away from zero; a carry into the exponent is the correct rounding), and the split
// inputs of both kernels are finite.  (A non-finite input gives a non-finite row either way.)
__device__ __forceinline__ void tf32_split(uint32_t x, uint32_t &hi, uint32_t &lo)
{
    hi = (x + 0x1000u) & 0xffffe000u;
    lo = __float_as_uint(__uint_as_float(x) - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float2 &c01, float2 &c23, const uint32_t a[4], uint32_t b0, uint32_t b1)
{
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(c01.x), "+f"(c01.y), "+f"(c23.x), "+f"(c23.y)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// C += A B in 3xTF32, always in this order (an output element then depends only on its own A row and the k order)
__device__ __forceinline__ void mma_3xtf32(float2 &c01, float2 &c23, const uint32_t ah[4], const uint32_t al[4], const float4 b)
{
    mma_tf32(c01, c23, al, __float_as_uint(b.x), __float_as_uint(b.y));
    mma_tf32(c01, c23, ah, __float_as_uint(b.z), __float_as_uint(b.w));
    mma_tf32(c01, c23, ah, __float_as_uint(b.x), __float_as_uint(b.y));
}
// ldmatrix of 32-bit elements: matrix i (8 rows of 16 bytes, row addresses from lanes 8i .. 8i+7) lands in r[i] as
// element (row lane >> 2, column lane & 3) -- an A fragment when the four matrices are (rows 0-7 | 8-15) x (k 0-3 | 4-7)
__device__ __forceinline__ void ldsm_x2(uint32_t saddr, uint32_t &r0, uint32_t &r1)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(saddr) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t saddr, uint32_t r[4])
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(saddr) : "memory");
}
// host side of the split: cvt.rna.tf32.f32 (nearest, ties away from zero)
static inline float tf32_rna_host(float x)
{
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) != 0x7f800000u) u = (u + 0x1000u) & 0xffffe000u;
    float r;
    memcpy(&r, &u, 4);
    return r;
}

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
