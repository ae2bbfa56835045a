// conv_l1.cu -- event-level Layer (conv_block1) of DAGR's backbone, sm_90a.
//
//   conv_a : SplineConv(3->16) + BN + act                      (conv.py:10-28)
//   conv_b : SplineConv(16->16) + BN, Linear(3->16)+BN skip, add, act   (conv.py:31-56)
//            fused with pool1's per-voxel channel max          (pooling.py:74-75)
//
// Formulation ("slot form" of MySplineConv.message_lut, spline_conv.py:39-47).  At the event level
// every edge offset is an integer pixel offset d in [-r,r]^2 and v = 4*attr lies in (1,3), so only
// 15 (3 in x, 5 in y) of the 5x5 spline kernels are reachable.  With tab[c][u] = LUT basis weight of
// slot u for spiral cell c:
//       A_u[i]  = sum_{e in N(i) + self}  tab[c_e][u] * x[src_e]          (phase 1, per edge)
//       out[i]  = sum_u  W_u^T A_u[i]  +  W_root^T x[i]                    (phase 2, per node)
// Phase-2 weights are uniform across lanes and are passed by value as a __grid_constant__ kernel
// parameter, so every FFMA takes its weight straight from the constant bank (no load instructions).
// One thread per destination node; nodes are in cell-major sorted order, so own rows, ELL columns
// and outputs are fully coalesced and the pool1 max is a warp-segmented reduction.
#include <string.h>
#include "common.cuh"

#define L1_THREADS 128

struct L1Smem {
    float *tab;     // [ncell][DAGR_TABW]
    float *posx;    // [W]
    float *posy;    // [H]
    short *sp;      // [ncell]
};

__device__ __forceinline__ L1Smem l1_smem_init(const dagr_geom_t &g, const float *__restrict__ tab, unsigned char *raw)
{
    L1Smem s;
    s.tab = (float *)raw;
    s.posx = s.tab + g.ncell * DAGR_TABW;
    s.posy = s.posx + g.W;
    s.sp = (short *)(s.posy + g.H);
    for (int i = threadIdx.x; i < g.ncell * DAGR_TABW; i += blockDim.x) s.tab[i] = tab[i];
    for (int i = threadIdx.x; i < g.W; i += blockDim.x) s.posx[i] = g.posx0[i];
    for (int i = threadIdx.x; i < g.H; i += blockDim.x) s.posy[i] = g.posy0[i];
    for (int i = threadIdx.x; i < g.ncell; i += blockDim.x)
        s.sp[i] = (short)(((int)g.spiral[2 * i] & 0xff) | ((int)g.spiral[2 * i + 1] << 8));
    __syncthreads();
    return s;
}

static size_t l1_smem_bytes(const dagr_geom_t *g)
{
    return (size_t)g->ncell * DAGR_TABW * 4 + (size_t)(g->W + g->H) * 4 + (size_t)g->ncell * 2 + 16;
}

__device__ __forceinline__ void load_tab(const float *row, float w[DAGR_KU])
{
    static_assert(DAGR_KU == 15 && DAGR_TABW == 16, "table row layout");
    const float4 a = *reinterpret_cast<const float4 *>(row);
    const float4 b = *reinterpret_cast<const float4 *>(row + 4);
    const float4 c = *reinterpret_cast<const float4 *>(row + 8);
    const float4 d = *reinterpret_cast<const float4 *>(row + 12);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
    w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
    w[8] = c.x; w[9] = c.y; w[10] = c.z; w[11] = c.w;
    w[12] = d.x; w[13] = d.y; w[14] = d.z;
}

// ------------------------------------------------------------------------------------------------
// conv_a
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(L1_THREADS)
k_l1_conv_a(const dagr_geom_t g, int64_t N, const uint32_t *__restrict__ xyb, const float *__restrict__ feat_s,
            const int32_t *__restrict__ nbr, const uint16_t *__restrict__ off, const float *__restrict__ tab,
            const __grid_constant__ dagr_l1a_params_t P, float *__restrict__ xa)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const L1Smem s = l1_smem_init(g, tab, smem_raw);
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;

    const uint32_t w = xyb[p];
    const int x = w & 0xfff, y = (w >> 12) & 0xfff;
    const float f0 = feat_s[p], f1 = s.posx[x], f2 = s.posy[y];
    const int n = nbr[(int64_t)(DAGR_ELL - 1) * N + p];

    float A[DAGR_KU][3];
    {
        float t[DAGR_KU];
        load_tab(s.tab, t);                                   // self loop: spiral cell 0, attr (0.5,0.5)
#pragma unroll
        for (int u = 0; u < DAGR_KU; u++) { A[u][0] = t[u] * f0; A[u][1] = t[u] * f1; A[u][2] = t[u] * f2; }
    }
    for (int q = 0; q < n; q++) {
        const int j = nbr[(int64_t)q * N + p];
        const int c = off[(int64_t)q * N + p];
        const int sp = s.sp[c];
        const float e0 = __ldg(feat_s + j);
        const float e1 = s.posx[x + (int)(signed char)(sp & 0xff)];
        const float e2 = s.posy[y + (sp >> 8)];
        float t[DAGR_KU];
        load_tab(s.tab + c * DAGR_TABW, t);
#pragma unroll
        for (int u = 0; u < DAGR_KU; u++) {
            A[u][0] = fmaf(t[u], e0, A[u][0]);
            A[u][1] = fmaf(t[u], e1, A[u][1]);
            A[u][2] = fmaf(t[u], e2, A[u][2]);
        }
    }
    float o[16];
#pragma unroll
    for (int k = 0; k < 16; k++) o[k] = 0.f;
#pragma unroll
    for (int u = 0; u < DAGR_KU; u++)
#pragma unroll
        for (int ci = 0; ci < 3; ci++)
#pragma unroll
            for (int k = 0; k < 16; k++) o[k] = fmaf(A[u][ci], P.w[u][ci][k], o[k]);
#pragma unroll
    for (int k = 0; k < 16; k++) {
        float r = o[k];
        r = fmaf(f0, P.root[0][k], r);
        r = fmaf(f1, P.root[1][k], r);
        r = fmaf(f2, P.root[2][k], r);
        r = fmaf(r, P.scale[k], P.shift[k]);
        o[k] = P.relu ? fmaxf(r, 0.f) : r;
    }
    // xa is stored half-major: [2][N][8] (channels 0-7, then 8-15), see conv_b v2
    const int sw = XA_SWZ(p);
    float4 *dst = reinterpret_cast<float4 *>(xa + p * 8);
    dst[sw] = make_float4(o[0], o[1], o[2], o[3]);
    dst[sw ^ 1] = make_float4(o[4], o[5], o[6], o[7]);
    dst = reinterpret_cast<float4 *>(xa + (N + p) * 8);
    dst[sw] = make_float4(o[8], o[9], o[10], o[11]);
    dst[sw ^ 1] = make_float4(o[12], o[13], o[14], o[15]);
}

extern "C" int dagr_l1_conv_a(const dagr_geom_t *g, int64_t N, const uint32_t *xyb, const float *feat_s,
                              const int32_t *nbr, const uint16_t *off, const float *tab,
                              const dagr_l1a_params_t *p_host, float *xa, void *stream)
{
    DAGR_CHECK_ARG(g && p_host, "null argument");
    if (N <= 0) return DAGR_OK;
    size_t smem = l1_smem_bytes(g);
    DAGR_CUDA(dagr_allow_smem(k_l1_conv_a, smem));
    k_l1_conv_a<<<dagr_div_up(N, L1_THREADS), L1_THREADS, smem, (cudaStream_t)stream>>>(
        *g, N, xyb, feat_s, nbr, off, tab, *p_host, xa);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// conv_b + skip + act + pool1 max
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(L1_THREADS)
k_l1_conv_b(const dagr_geom_t g, int64_t N, const uint32_t *__restrict__ xyb, const float *__restrict__ feat_s,
            const float *__restrict__ xa, const int32_t *__restrict__ nbr, const uint16_t *__restrict__ off,
            const float *__restrict__ tab, const __grid_constant__ dagr_l1b_params_t P,
            float *__restrict__ x1, uint32_t *__restrict__ poolmax)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const L1Smem s = l1_smem_init(g, tab, smem_raw);
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = p < N;
    float o[16];
#pragma unroll
    for (int k = 0; k < 16; k++) o[k] = 0.f;
    int cell = -1;
    if (active) {
        const uint32_t w = xyb[p];
        const int x = w & 0xfff, y = (w >> 12) & 0xfff, b = w >> 24;
        cell = b * (g.ny1 * g.nx1) + (__ldg(g.ykey + y) / (g.nx1 * g.CP)) * g.nx1 + __ldg(g.xkey + x) / g.CP;
        const int n = nbr[(int64_t)(DAGR_ELL - 1) * N + p];

        // Two passes over the input-channel halves keep the slot accumulators A[15][8] in registers
        // (15 of the 25 spline kernels are reachable: 3 in x, 5 in y because attr_y is normalised by H).
#pragma unroll 1
        for (int half = 0; half < 2; half++) {
            float2 A[DAGR_KU][4];
            {
                // self loop (spiral cell 0) and root weight: own row
                const float4 *src = reinterpret_cast<const float4 *>(xa + ((int64_t)half * N + p) * 8);
                const float4 t0 = src[XA_SWZ(p)], t1 = src[XA_SWZ(p) ^ 1];
                const float2 v[4] = {make_float2(t0.x, t0.y), make_float2(t0.z, t0.w), make_float2(t1.x, t1.y), make_float2(t1.z, t1.w)};
                float t[DAGR_KU];
                load_tab(s.tab, t);
#pragma unroll
                for (int u = 0; u < DAGR_KU; u++)
#pragma unroll
                    for (int k = 0; k < 4; k++) A[u][k] = make_float2(t[u] * v[k].x, t[u] * v[k].y);
                if (half == 0) {
#pragma unroll
                    for (int k = 0; k < 4; k++)
#pragma unroll
                        for (int c = 0; c < 16; c++) {
                            o[c] = fmaf(v[k].x, P.root[2 * k][c], o[c]);
                            o[c] = fmaf(v[k].y, P.root[2 * k + 1][c], o[c]);
                        }
                } else {
#pragma unroll
                    for (int k = 0; k < 4; k++)
#pragma unroll
                        for (int c = 0; c < 16; c++) {
                            o[c] = fmaf(v[k].x, P.root[8 + 2 * k][c], o[c]);
                            o[c] = fmaf(v[k].y, P.root[8 + 2 * k + 1][c], o[c]);
                        }
                }
            }
            // phase 1: gather neighbours
            for (int q = 0; q < n; q++) {
                const int j = nbr[(int64_t)q * N + p];
                const int c = off[(int64_t)q * N + p];
                const float4 *src = reinterpret_cast<const float4 *>(xa + ((int64_t)half * N + j) * 8);
                const float4 t0 = __ldg(src + XA_SWZ(j)), t1 = __ldg(src + (XA_SWZ(j) ^ 1));
                const float2 e[4] = {make_float2(t0.x, t0.y), make_float2(t0.z, t0.w), make_float2(t1.x, t1.y), make_float2(t1.z, t1.w)};
                float t[DAGR_KU];
                load_tab(s.tab + c * DAGR_TABW, t);
#pragma unroll
                for (int u = 0; u < DAGR_KU; u++) {
                    const float2 tt = make_float2(t[u], t[u]);
#pragma unroll
                    for (int k = 0; k < 4; k++) A[u][k] = ffma2(tt, e[k], A[u][k]);
                }
            }
            // phase 2: o += sum_u W_u^T A_u   (weights from the constant bank, uniform across the warp)
            if (half == 0) {
#pragma unroll
                for (int u = 0; u < DAGR_KU; u++)
#pragma unroll
                    for (int k = 0; k < 4; k++)
#pragma unroll
                        for (int c = 0; c < 16; c++) {
                            o[c] = fmaf(A[u][k].x, P.w[u][2 * k][c], o[c]);
                            o[c] = fmaf(A[u][k].y, P.w[u][2 * k + 1][c], o[c]);
                        }
            } else {
#pragma unroll
                for (int u = 0; u < DAGR_KU; u++)
#pragma unroll
                    for (int k = 0; k < 4; k++)
#pragma unroll
                        for (int c = 0; c < 16; c++) {
                            o[c] = fmaf(A[u][k].x, P.w[u][8 + 2 * k][c], o[c]);
                            o[c] = fmaf(A[u][k].y, P.w[u][8 + 2 * k + 1][c], o[c]);
                        }
            }
        }
        // BN, skip branch BN(Linear(x0)), add, act  (conv.py:47-56)
        const float f0 = feat_s[p], f1 = s.posx[x], f2 = s.posy[y];
#pragma unroll
        for (int c = 0; c < 16; c++) {
            float sk = f0 * P.skip[0][c];
            sk = fmaf(f1, P.skip[1][c], sk);
            sk = fmaf(f2, P.skip[2][c], sk);
            sk = fmaf(sk, P.sscale[c], P.sshift[c]);
            float r = fmaf(o[c], P.scale[c], P.shift[c]) + sk;
            o[c] = P.relu ? fmaxf(r, 0.f) : r;
        }
        if (x1 != nullptr) {
            float4 *dst = reinterpret_cast<float4 *>(x1 + p * 16);
            dst[0] = make_float4(o[0], o[1], o[2], o[3]);
            dst[1] = make_float4(o[4], o[5], o[6], o[7]);
            dst[2] = make_float4(o[8], o[9], o[10], o[11]);
            dst[3] = make_float4(o[12], o[13], o[14], o[15]);
        }
    }
    // pool1 max: nodes of one voxel are contiguous -> warp-segmented max, heads publish with atomicMax
    if (poolmax != nullptr) {
        const int lane = threadIdx.x & 31;
        uint32_t eo[16];
#pragma unroll
        for (int c = 0; c < 16; c++) eo[c] = active ? enc_ordered(o[c]) : 0u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int oc = __shfl_down_sync(0xffffffffu, cell, d);
            const bool take = (lane + d < 32) && (oc == cell);
#pragma unroll
            for (int c = 0; c < 16; c++) {
                const uint32_t ov = __shfl_down_sync(0xffffffffu, eo[c], d);
                if (take) eo[c] = max(eo[c], ov);
            }
        }
        const int pc = __shfl_up_sync(0xffffffffu, cell, 1);
        const bool head = active && (lane == 0 || pc != cell);
        if (head) {
            uint32_t *dst = poolmax + (int64_t)cell * 16;
#pragma unroll
            for (int c = 0; c < 16; c++) atomicMax(dst + c, eo[c]);
        }
    }
}

extern "C" int dagr_l1_conv_b_pool(const dagr_geom_t *g, int64_t N, const uint32_t *xyb, const float *feat_s,
                                   const float *xa, const int32_t *nbr, const uint16_t *off, const float *tab,
                                   const dagr_l1b_params_t *p_host, float *x1, uint32_t *poolmax, void *stream)
{
    DAGR_CHECK_ARG(g && p_host, "null argument");
    DAGR_CHECK_ARG(p_host->pool_mean == 0, "mean pooling needs the per-voxel kernel (dagr_l1_conv_b_pool_voxel)");
    if (N <= 0) return DAGR_OK;
    size_t smem = l1_smem_bytes(g);
    DAGR_CUDA(dagr_allow_smem(k_l1_conv_b, smem));
    k_l1_conv_b<<<dagr_div_up(N, L1_THREADS), L1_THREADS, smem, (cudaStream_t)stream>>>(
        *g, N, xyb, feat_s, xa, nbr, off, tab, *p_host, x1, poolmax);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ================================================================================================
// conv_b v2: one CTA per pool1 voxel, neighbour rows staged in shared memory by TMA bulk copies
// ================================================================================================
// Because nodes are stored in cell-major order, the xa rows any node of the voxel can gather are the
// rows of its 3x3 voxel neighbourhood = THREE contiguous runs.  One elected thread issues three
// cp.async.bulk (TMA, 1-D) copies global -> shared that complete on an mbarrier; all gathers of phase 1
// then hit shared memory.  The per-voxel channel max, mean position and pixel rounding of pool1
// (pooling.py:66-86) are finished in the same CTA, so neither the per-node activations nor a separate
// finalize pass touch HBM.  Voxels whose neighbourhood exceeds the staging buffer gather from global.
// Two instances (template parameters CAP = staged half-rows of 32 B, THREADS = CTA size), like the build kernel:
//   regular : one CTA per voxel, 160 threads, 1344 rows (43 KB), 4 CTAs per SM;
//   dense   : voxels whose 3x3 neighbourhood holds more rows (75 % of the events of the clustered benchmark stream) are
//             queued by the regular kernel and processed by persistent 384-thread CTAs (one per SM) that stage up to
//             6144 rows (196 KB); only beyond that rows are gathered from global memory / L2.
#define CB2_THREADS 160
#define CB2_CAP 1344
#define CB2_THREADS_BIG 384
#define CB2_CAP_BIG 6144
static_assert(2 * CB2_CAP_BIG <= 16384, "the ELL word keeps 2*row+swizzle in 14 bits");
#define CB2_G 5                  // spline slots per pass: one x-slot k, all five y-slots (u = k + 3 j)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

struct CB2Tile {
    int run_start[3], run_len[3], run_off[3];
};

// ---- phase 2 on tensor cores (CB2_TC = 1) ------------------------------------------------------------------------------
// Phase 2 of a pass is a dense product with node-independent weights, [32 nodes of a warp x 40] x [40 x 16]: on CUDA cores it
// costs as many issue slots as the edge loop (every FFMA needs its weight through a uniform constant load on sm_90).  With
// CB2_TC it runs as mma.sync.m16n8k8 TF32 in 3xTF32 form (a_hi*b_hi + a_hi*b_lo + a_lo*b_hi, hi = cvt.rna.tf32(x),
// lo = x - hi; relative error ~1e-6): the warp's 32 nodes are two m16 tiles, the 16 outputs two n8 tiles, one k8 step per
// spline slot (8 channels of the current half) plus one per half for the root weight.  o2[8] then holds the FP32 C fragments
// across all passes: o2[4 mt + 2 nt] = (c0, c1), o2[4 mt + 2 nt + 1] = (c2, c3) of m-tile mt, n-tile nt.  An output element
// depends only on its own node's row and the fixed k order, so a node gets the same bits in every instance and CTA shape.
// The weight fragments (per lane, already split into hi / lo) come from global memory in the order of dagr_l1_tc_weights:
// float4 [half][k-step: slot 0..14, root = 15][lane][n-tile] = (hi k=t, hi k=t+4, lo k=t, lo k=t+4), t = lane & 3.
// Phase 1 leaves one node per lane; the A fragment needs other lanes' values, which go through a 256-byte per-warp tile
// (16 rows x 4 floats: one m-tile and half a k-step at a time, so that four CTAs still fit an SM).
#ifndef CB2_TC
#define CB2_TC 1
#endif
#define CB2_TC_KSTEPS 16                   // per channel half: 15 spline slots + root

// o2 (C fragments) += [this warp's nodes x 8] x [8 x 16]; this lane's node contributes a[0..7], wf = this k-step's fragments
// of this lane.  Warp-uniform call; lanes without a node pass zeros.  (tf32_split / mma_3xtf32 / ldsm_*: common.cuh)
__device__ __forceinline__ void cb2_tc_kstep(float *xt, const float a[8], const float4 *__restrict__ wf, float2 o2[8])
{
    const int lane = threadIdx.x & 31;
    const float4 w0 = __ldg(wf), w1 = __ldg(wf + 1);
    const uint32_t bh[2][2] = {{__float_as_uint(w0.x), __float_as_uint(w0.y)}, {__float_as_uint(w1.x), __float_as_uint(w1.y)}};
    const uint32_t bl[2][2] = {{__float_as_uint(w0.z), __float_as_uint(w0.w)}, {__float_as_uint(w1.z), __float_as_uint(w1.w)}};
    float *row = xt + 4 * (lane & 15);
    const uint32_t ra = smem_u32(row);
#pragma unroll
    for (int mt = 0; mt < 2; mt++) {
        uint32_t ah[4], al[4];
#pragma unroll
        for (int h = 0; h < 2; h++) {                              // k = 4h .. 4h+3 of rows 16mt .. 16mt+15
            __syncwarp();
            if ((lane >> 4) == mt) *reinterpret_cast<float4 *>(row) = make_float4(a[4 * h], a[4 * h + 1], a[4 * h + 2], a[4 * h + 3]);
            __syncwarp();
            uint32_t r0, r1;                                       // r0 = A[g][4h + t], r1 = A[g + 8][4h + t]
            ldsm_x2(ra, r0, r1);
            tf32_split(r0, ah[2 * h], al[2 * h]);
            tf32_split(r1, ah[2 * h + 1], al[2 * h + 1]);
        }
        // (a0, a1, a2, a3) = (A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4]): the order of ah / al above
        const uint32_t fa[4] = {ah[0], ah[1], ah[2], ah[3]}, fl[4] = {al[0], al[1], al[2], al[3]};
#pragma unroll
        for (int nt = 0; nt < 2; nt++) {                           // the 3xTF32 order of mma_3xtf32
            mma_tf32(o2[4 * mt + 2 * nt], o2[4 * mt + 2 * nt + 1], fl, bh[nt][0], bh[nt][1]);
            mma_tf32(o2[4 * mt + 2 * nt], o2[4 * mt + 2 * nt + 1], fa, bl[nt][0], bl[nt][1]);
            mma_tf32(o2[4 * mt + 2 * nt], o2[4 * mt + 2 * nt + 1], fa, bh[nt][0], bh[nt][1]);
        }
    }
}

// C fragments -> thread-per-node layout (o2[c] = channels 2c, 2c+1 of this lane's node), through the same tile.  Warp-uniform.
__device__ __forceinline__ void cb2_tc_unfrag(float *xt, float2 o2[8])
{
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    float2 r[8];
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
        for (int q = 0; q < 4; q++) {                              // channels 4q .. 4q+3 = n-tile q/2, lanes with t/2 == q%2
            __syncwarp();
            if ((t >> 1) == (q & 1)) {
                *reinterpret_cast<float2 *>(xt + 4 * g + 2 * (t & 1)) = o2[4 * mt + 2 * (q >> 1)];
                *reinterpret_cast<float2 *>(xt + 4 * (g + 8) + 2 * (t & 1)) = o2[4 * mt + 2 * (q >> 1) + 1];
            }
            __syncwarp();
            const float4 v = *reinterpret_cast<const float4 *>(xt + 4 * (lane & 15));
            if ((lane >> 4) == mt) { r[2 * q] = make_float2(v.x, v.y); r[2 * q + 1] = make_float2(v.z, v.w); }
        }
#pragma unroll
    for (int c = 0; c < 8; c++) o2[c] = r[c];
}

// One pass = one input-channel half (8 channels) x one x-slot k (the 5 spline slots u = k + 3 j, j = 0..4) of one node:
//     A_j = sum_{e in N(i) + self} tabx[dx_e][k] * taby[dy_e][j] * x_e[half]      (5 x 8 accumulators)
//     o  += sum_j W_{k+3j}[half]^T A_j
// The slot weights are rebuilt from the two per-axis factor tables (2r+1 rows each, geometry.py) instead of a
// [ncell][16] table: 1.5 KB instead of 21 KB of shared memory per CTA, which is what lets four CTAs share an SM.
// `half` and `k` are template parameters so the phase-2 weights come through the uniform datapath (LDCU.128);
// a run-time pass index makes ptxas fetch them with register-indexed LDC, which saturates the ADU pipe.
// s_ell[q][tid]: see the staged loop below (byte offsets of the row chunks and of the two factor-table rows).
// Variants measured and rejected (ELL entries ordered by the x-slots they feed so that the outer x-slot passes skip their
// exact-zero edges: slower, the per-lane loop bounds cost more than the skipped iterations save): 15 slots x 8 channels per pass (120
// accumulators, 2 CTAs/SM), 15 slots x 4 channels, phase-2 weights from shared memory or half/half.
// With TC, phase 2 runs on tensor cores (see cb2_tc_kstep) and o2 holds C fragments; the call is then warp-uniform and a lane
// without a node passes n = -1 (no edge, A = 0).
template <bool STAGED, int half, int grp, int THREADS, bool TC, class PT>
__device__ __forceinline__ void cb2_pass(int64_t N, int p, int n, const float *__restrict__ xa, const float *s_rows,
                                         const float *s_wx, const float4 *s_wy, const float *s_wy4, const uint32_t *s_ell, const uint16_t *s_sp,
                                         const int32_t *__restrict__ nbr, const uint16_t *__restrict__ off,
                                         const PT &P, const float4 *__restrict__ wfrag, float *xt, int own_row, int r, int tix, float2 o2[8])
{
    float2 A[CB2_G][4];
#pragma unroll
    for (int u = 0; u < CB2_G; u++)
#pragma unroll
        for (int k = 0; k < 4; k++) A[u][k] = make_float2(0.f, 0.f);
#define CB2_EDGE_FMA()                                                                                              \
    do {                                                                                                            \
        const float2 e[4] = {make_float2(t0.x, t0.y), make_float2(t0.z, t0.w), make_float2(t1.x, t1.y), make_float2(t1.z, t1.w)}; \
        const float wy[CB2_G] = {wya.x, wya.y, wya.z, wya.w, wy4};                                                  \
        _Pragma("unroll") for (int j = 0; j < CB2_G; j++) {                                                         \
            const float w = __fmul_rn(wy[j], wx);           /* == tab[c][grp + 3 j] bit for bit (geometry.py) */    \
            const float2 tt = make_float2(w, w);                                                                    \
            _Pragma("unroll") for (int k = 0; k < 4; k++) A[j][k] = ffma2(tt, e[k], A[j][k]);                       \
        }                                                                                                           \
    } while (0)
    if constexpr (STAGED) {
        // the ELL word carries ready-made BYTE offsets: bits 4..17 = 16 * (2 * row + row swizzle) (first 16-byte chunk of
        // the staged half-row; the other chunk is that offset ^ 16), bits 18..22 = dx + r, bits 23..27 = dy + r.  Slot 0 is
        // the self loop.  Every instruction costs an issue slot (one per cycle and SMSP) and the loop is issue bound, so
        // saving these 8 shifts/masks/adds per edge and pass is worth it.
        const char *rb = reinterpret_cast<const char *>(s_rows);
        // factor tables, laid out so that a warp's lookups do not collide: wx [3 x-slots][32 offsets] (stride 4 B: lanes with the
        // same offset broadcast, different offsets hit different banks), wy[0..3] as one float4 per offset (16 B stride), wy[4] apart
        const char *wxb = reinterpret_cast<const char *>(s_wx) + 128 * grp, *wyb = reinterpret_cast<const char *>(s_wy);
        const char *wy4b = reinterpret_cast<const char *>(s_wy4);
#ifndef CB2_UNROLL
#define CB2_UNROLL 1                                                    // measured: every larger unroll is slower (registers, I-cache)
#endif
        constexpr int kUnroll = CB2_UNROLL;
        // (most of this kernel's stall samples are short-scoreboard waits on this loop's shared-memory loads -- ELL word -> row
        // address -> row is a chain of two dependent loads per edge.  Software prefetching was measured in a same-box A/B:
        // next edge's ELL word one iteration ahead, or the next edge's row and table entries as well: both slower.)
#pragma unroll kUnroll
        for (int q = 0; q <= n; q++) {
            const uint32_t ell = s_ell[q * THREADS + tix];
            const uint32_t ro = ell & 0x3fff0u, xo = (ell >> 16) & 0x7cu, yo = (ell >> 19) & 0x1f0u;
            const float4 t0 = *reinterpret_cast<const float4 *>(rb + ro), t1 = *reinterpret_cast<const float4 *>(rb + (ro ^ 16u));
            const float wx = *reinterpret_cast<const float *>(wxb + xo);
            const float4 wya = *reinterpret_cast<const float4 *>(wyb + yo);
            const float wy4 = *reinterpret_cast<const float *>(wy4b + (yo >> 2));
            CB2_EDGE_FMA();
        }
    } else {
#pragma unroll 1
        for (int q = -1; q < n; q++) {                                   // q = -1: self loop (offset 0,0)
            int row, dxi, dyi;
            if (q < 0) { row = p; dxi = r; dyi = r; }
            else {
                row = nbr[(int64_t)q * N + p];
                const uint32_t d = s_sp[off[(int64_t)q * N + p]];
                dxi = (int)(d & 31u); dyi = (int)(d >> 5);
            }
            const int sw = XA_SWZ(row);
            const float4 *src = reinterpret_cast<const float4 *>(xa + ((int64_t)half * N + row) * 8);
            const float4 t0 = src[sw], t1 = src[sw ^ 1];
            const float wx = s_wx[grp * 32 + dxi];
            const float4 wya = s_wy[dyi];
            const float wy4 = s_wy4[dyi];
            CB2_EDGE_FMA();
        }
    }
#undef CB2_EDGE_FMA
    if constexpr (TC) {
        // phase 2 on tensor cores: k-step j = spline slot grp + 3 j, k = channel of this half
        // The pass sums into fresh fragments which are then added to o2 with IEEE fp32 adds: the tensor cores' fp32
        // accumulation truncates, and chaining all 6 passes x 15 mma through it doubled the largest errors against the oracle.
        const float4 *wf = wfrag + ((size_t)half * CB2_TC_KSTEPS * 32 + (threadIdx.x & 31)) * 2;
        float2 c2[8];
#pragma unroll
        for (int i = 0; i < 8; i++) c2[i] = make_float2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < CB2_G; j++) {
            const float a[8] = {A[j][0].x, A[j][0].y, A[j][1].x, A[j][1].y, A[j][2].x, A[j][2].y, A[j][3].x, A[j][3].y};
            cb2_tc_kstep(xt, a, wf + (grp + 3 * j) * 64, c2);
        }
#pragma unroll
        for (int i = 0; i < 8; i++) o2[i] = make_float2(__fadd_rn(o2[i].x, c2[i].x), __fadd_rn(o2[i].y, c2[i].y));
        return;
    }
    // phase 2: weights from the constant bank through uniform 128-bit loads, two FFMA2 per load
#pragma unroll
    for (int j = 0; j < CB2_G; j++)
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int c4 = 0; c4 < 4; c4++) {
                const float4 wa = *reinterpret_cast<const float4 *>(&P.w[grp + 3 * j][8 * half + 2 * k][4 * c4]);
                const float4 wb = *reinterpret_cast<const float4 *>(&P.w[grp + 3 * j][8 * half + 2 * k + 1][4 * c4]);
                o2[2 * c4] = ffma2(make_float2(A[j][k].x, A[j][k].x), make_float2(wa.x, wa.y), o2[2 * c4]);
                o2[2 * c4 + 1] = ffma2(make_float2(A[j][k].x, A[j][k].x), make_float2(wa.z, wa.w), o2[2 * c4 + 1]);
                o2[2 * c4] = ffma2(make_float2(A[j][k].y, A[j][k].y), make_float2(wb.x, wb.y), o2[2 * c4]);
                o2[2 * c4 + 1] = ffma2(make_float2(A[j][k].y, A[j][k].y), make_float2(wb.z, wb.w), o2[2 * c4 + 1]);
            }
}

__device__ __forceinline__ float cb2_div_floor(float a, float b)
{
    const float mod = fmodf(a, b);
    float div = __fdiv_rn(__fsub_rn(a, mod), b);
    if ((mod != 0.f) && ((b < 0.f) != (mod < 0.f))) div -= 1.f;
    float fl;
    if (div != 0.f) { fl = floorf(div); if (div - fl > 0.5f) fl += 1.f; }
    else fl = copysignf(0.f, __fdiv_rn(a, b));
    return fl;
}
__device__ __forceinline__ int cb2_round_to_pixel(float mean, int size)
{
    const float inv = __frcp_rn((float)size);
    const int k = (int)cb2_div_floor(__fadd_rn(mean, 1e-5f), inv);
    return min(max(k, 0), size - 1);
}

// The kernel is a template over the input rows: <dagr_l1b_params_t, 2, false> is conv_block2 (16 channels = 2 staged
// 8-channel chunks, skip + act + pool1 epilogue); <dagr_l1img_params_t, 3, true> is the image-fusion variant of
// conv_block1.conv_block1 (the 16 sampled image channels = 2 chunks, added to the (polarity, x, y) part the probe kernel
// already summed; epilogue = BN + act, rows written back
// chunk-major for conv_block2, plus the layer's skip branch BN(Linear(x0)) -> skip_out; no pooling).
template <int THREADS>
struct CB2Shared {
    CB2Tile T;
    uint64_t bar;
    float red[THREADS / 32][16];
    long long sum[THREADS / 32][3];
    int tm[THREADS / 32];
    __align__(16) float xt[THREADS / 32][64];   // per-warp exchange tile of the tensor-core phase 2
};

// The per-voxel routine is a template over the input rows: <dagr_l1b_params_t, 2, false> is conv_block2 (16 channels = 2
// staged 8-channel chunks, skip + act + pool1 epilogue); <dagr_l1img_params_t, 3, true> is the image-fusion variant of
// conv_block1.conv_block1 (the 16 sampled image channels = 2 chunks, added to the (polarity, x, y) part the probe kernel
// already summed; epilogue = BN + act, rows written back
// chunk-major for conv_block2, plus the layer's skip branch BN(Linear(x0)) -> skip_out; no pooling).
// work list: wl_hdr[0] = number of voxels beyond this instance's staging capacity (queued in wl_ids when `defer`, otherwise
// only counted and gathered from global memory / L2), wl_hdr[1] = pop cursor of the dense kernel
template <class PT, int NCH, bool MODE_A, int CAP, int THREADS, bool POOL_MEAN, bool PLAIN, bool TC>
__device__ __forceinline__ void cb2_voxel(const dagr_geom_t &g, int64_t N, const int32_t *__restrict__ start, const uint32_t *__restrict__ xyb,
             const int2 *__restrict__ ti, const float *__restrict__ feat_s, const float *__restrict__ xa,
             const int32_t *__restrict__ nbr, const uint16_t *__restrict__ off,
             const PT &P, const float4 *__restrict__ wfrag, const float *__restrict__ skip_pre_in, const int min_idx_in,
             float *__restrict__ persist_in, float *__restrict__ x1_in, int32_t *__restrict__ cnt, int32_t *__restrict__ pxy,
             float *__restrict__ tmean, float *__restrict__ tmax, float *__restrict__ xg, int ldx,
             float *__restrict__ xa_out, float *__restrict__ skip_out,
             const int cell, unsigned char *smem_raw, CB2Shared<THREADS> &S, uint32_t &parity,
             int32_t *__restrict__ wl_hdr, int32_t *__restrict__ wl_ids, const int defer)
{
    // PLAIN = the synchronous events-only forward (no incremental mode, no running stream max, no per-node output, skip branch
    // computed here, ReLU): with these known at compile time the max instance is faster (A/B on one GPU)
    const int min_idx = PLAIN ? 0 : min_idx_in;
    float *const persist = PLAIN ? nullptr : persist_in;
    float *const x1 = PLAIN ? nullptr : x1_in;
    const float *const skip_pre = PLAIN ? nullptr : skip_pre_in;
    const bool relu = PLAIN ? true : (P.relu != 0);
    CB2Tile &T = S.T;
    uint64_t &s_bar = S.bar;
    auto &s_red = S.red;
    auto &s_sum = S.sum;
    auto &s_tm = S.tm;
    float *const xt = S.xt[threadIdx.x >> 5];
    float *s_rows = (float *)smem_raw;                                  // [CAP][8]   one channel half of the 3 runs
    float *s_wx = s_rows + (size_t)CAP * 8;                              // [3][32]   x factor of the slot weights, per x-slot
    float4 *s_wy = (float4 *)(s_wx + 128);                               // [32]      y factors 0..3
    float *s_wy4 = (float *)(s_wy + 32);                                 // [32]      y factor 4
    uint32_t *s_ell = (uint32_t *)(s_wy + 64);                           // [16][THREADS]  slot 0 = self loop (384 floats of tables before it)
    uint16_t *s_sp = (uint16_t *)(s_ell + DAGR_ELL * THREADS);           // [ncell]  (dx + r) | (dy + r) << 5
    const int per = g.ny1 * g.nx1;
    const int b = cell / per, rem = cell % per, cy = rem / g.nx1, cx = rem % g.nx1;
    const int p0 = start[(int64_t)cell * g.CP], p1 = start[(int64_t)(cell + 1) * g.CP];
    const int nown = p1 - p0;
    if (nown == 0) {                                                     // block-uniform
        if (MODE_A) return;
        if (threadIdx.x == 0) { cnt[cell] = 0; pxy[2 * cell] = 0; pxy[2 * cell + 1] = 0; tmean[cell] = 0.f; tmax[cell] = 0.f; }
        if (threadIdx.x < 16) xg[(int64_t)cell * ldx + threadIdx.x] = 0.f;
        return;
    }
    if (threadIdx.x < 32) {
        // the six run boundaries are independent loads: one lane each, then lane 0 lays the runs out
        const int clo = max(cx - 1, 0), chi = min(cx + 1, g.nx1 - 1);
        const int lane = threadIdx.x, rr = lane >> 1, ry = cy - 1 + rr;
        int v = 0;
        if (lane < 6 && ry >= 0 && ry < g.ny1)
            v = start[((int64_t)b * per + ry * g.nx1 + ((lane & 1) ? chi + 1 : clo)) * g.CP];
        int o = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int s0 = __shfl_sync(0xffffffffu, v, 2 * k), e0 = __shfl_sync(0xffffffffu, v, 2 * k + 1);
            const bool ok = (cy - 1 + k >= 0) && (cy - 1 + k < g.ny1);
            if (lane == 0) { T.run_start[k] = ok ? s0 : 0; T.run_len[k] = ok ? e0 - s0 : 0; T.run_off[k] = o; }
            o += ok ? e0 - s0 : 0;
        }
    }
    for (int i = threadIdx.x; i < 2 * g.r + 1; i += blockDim.x) {
        const float4 tx = __ldg(reinterpret_cast<const float4 *>(g.tabx) + i);
        s_wx[i] = tx.x; s_wx[32 + i] = tx.y; s_wx[64 + i] = tx.z;
        s_wy[i] = __ldg(reinterpret_cast<const float4 *>(g.taby) + 2 * i);
        s_wy4[i] = __ldg(g.taby + 8 * i + 4);
    }
    for (int i = threadIdx.x; i < g.ncell; i += blockDim.x)
        s_sp[i] = (uint16_t)(((int)g.spiral[2 * i] + g.r) | (((int)g.spiral[2 * i + 1] + g.r) << 5));
    __syncthreads();
    const int total = T.run_off[2] + T.run_len[2];
    const bool staged = total <= CAP;                                    // block-uniform
    if (!staged && wl_hdr != nullptr) {
        // more rows than this instance can stage: queue the voxel for the dense kernel (next launch on the stream) -- or,
        // when the caller did not ask for that, just count it
        int slot = 0;
        if (threadIdx.x == 0) slot = atomicAdd(&wl_hdr[0], 1);
        if (defer) { if (threadIdx.x == 0) wl_ids[slot] = cell; return; }
    }
    const int s1 = T.run_start[1];
    const int s2 = T.run_len[2] > 0 ? T.run_start[2] : 0x7fffffff;
    const int d0 = T.run_off[0] - T.run_start[0], d1 = T.run_off[1] - T.run_start[1], d2 = T.run_off[2] - T.run_start[2];

    // pool1 aggregation (pooling.py:74-77).  A template parameter: as a run-time flag (selects in the row epilogue and in the
    // reductions, one more live predicate) it slowed the max instance down (A/B on one GPU)
    constexpr bool pool_mean = POOL_MEAN && !MODE_A;
    float m[16];
#pragma unroll
    for (int c = 0; c < 16; c++) m[c] = pool_mean ? 0.f : -INFINITY;
    long long sx = 0, sy = 0, st = 0;
    int tm = -2147483647;
    // Sparse voxels (at most one warp of nodes, e.g. the early windows of an inter-frame sequence): the per-thread chain of
    // six passes is the whole run time of the CTA and four of its five warps would idle.  Warps 0..2 then share the SAME
    // nodes and take one x-slot each (both channel halves), their partial sums are added through shared memory: a third of
    // the serial work per thread.  Block-uniform; the dense path below is unchanged.
    // (compiled into the image-fusion instance only: in the 2-chunk conv_block2 instance the extra live state costs the
    // dense path 1.3 % and the sparse gain is small, measured).  Incremental steps take the same path, so that a new node gets
    // the bits the synchronous forward gives it (the passes skip the nodes that are not active).
    const bool sparse = MODE_A && staged && nown <= 32;
    const int lane_ = threadIdx.x & 31, wid_ = threadIdx.x >> 5;
    for (int pb0 = p0; pb0 < p1; pb0 += blockDim.x) {
        const int p = sparse ? p0 + lane_ : pb0 + threadIdx.x;
        const bool inrange = sparse ? (p < p1 && wid_ < 3) : (p < p1);
        const int tix = sparse ? lane_ : (int)threadIdx.x;                // column of this node in s_ell
        // incremental mode: only new nodes are convolved (the arrival index is only looked at then)
        const bool active = inrange && (min_idx <= 0 || ti[p].y >= min_idx);
        if (min_idx > 0 && !__syncthreads_or(active)) {                  // block-uniform: nothing new in this chunk
            if (inrange) { const uint32_t w0 = xyb[p]; const int t0 = ti[p].x; sx += w0 & 0xfff; sy += (w0 >> 12) & 0xfff; st += t0; tm = max(tm, t0); }
            continue;
        }
        const int n = active ? nbr[(int64_t)(DAGR_ELL - 1) * N + p] : 0;
        // stage this node's ELL row (independent loads -> one global latency); neighbour positions become staged rows
        if (staged && active && (!sparse || wid_ == 0)) {
            int jj[DAGR_ELL - 1]; int cc[DAGR_ELL - 1];
#pragma unroll
            for (int q = 0; q < DAGR_ELL - 1; q++) {
                jj[q] = (q < n) ? nbr[(int64_t)q * N + p] : 0;
                cc[q] = (q < n) ? (int)off[(int64_t)q * N + p] : 0;
            }
#pragma unroll
            for (int q = 0; q < DAGR_ELL - 1; q++) {
                const int j = jj[q];
                const int row = j + (j >= s2 ? d2 : (j >= s1 ? d1 : d0));
                s_ell[(q + 1) * THREADS + tix] = ((uint32_t)(2 * row + XA_SWZ(j)) << 4) | ((uint32_t)s_sp[cc[q]] << 18);
            }
            s_ell[tix] = ((uint32_t)(2 * (p + d1) + XA_SWZ(p)) << 4) | ((uint32_t)(g.r | (g.r << 5)) << 18);   // self loop
        }
        float2 o2[8], sk2[MODE_A ? 8 : 1];
#pragma unroll
        for (int k = 0; k < 8; k++) o2[k] = make_float2(0.f, 0.f);
#pragma unroll
        for (int k = 0; k < (MODE_A ? 8 : 1); k++) sk2[k] = make_float2(0.f, 0.f);
#pragma unroll 1
        for (int half = 0; half < NCH; half++) {
            if (staged) {
                __syncthreads();                                        // everyone is done with the previous half's rows
                if (threadIdx.x == 0) {
                    // TMA: three contiguous runs of 32-byte half-rows, global -> shared, completion on the mbarrier
                    // (issuing the first half during the CTA's set-up, so that it flies while the tables and ELL rows are
                    // fetched, was measured and gave nothing; the other three CTAs of the SM already hide that latency)
                    mbar_expect_tx(&s_bar, (uint32_t)total * 32u);
                    for (int rr = 0; rr < 3; rr++)
                        if (T.run_len[rr] > 0)
                            tma_bulk_g2s(s_rows + (size_t)T.run_off[rr] * 8, xa + ((size_t)half * N + T.run_start[rr]) * 8,
                                         (uint32_t)T.run_len[rr] * 32u, &s_bar);
                }
                mbar_wait(&s_bar, parity);                              // (one waiting thread + a CTA barrier instead: slower)
                parity ^= 1;
            }
            // with TC the warp's lanes run the passes together (mma.sync): a lane without a node joins with no edges
            if (TC ? __any_sync(0xffffffffu, active) : active) {
                const int nn = active ? n : -1;
                // root weight on this half of x_i.  `half` must be a compile-time constant here as well: with a run-time index
                // the 64 weight fetches per half become register-indexed LDC through the address-divergence unit
#define CB2_ROOT(H)                                                                                                  \
    do {                                                                                                            \
        const float4 *src = staged ? reinterpret_cast<const float4 *>(s_rows + (int64_t)(p + d1) * 8)               \
                                   : reinterpret_cast<const float4 *>(xa + ((int64_t)(H) * N + p) * 8);             \
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);                                                         \
        const float4 t0 = active ? src[XA_SWZ(p)] : z4, t1 = active ? src[XA_SWZ(p) ^ 1] : z4;                      \
        const float v[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};                                        \
        if constexpr (TC) {                                                                                         \
            float2 c2[8];                                                                                           \
            _Pragma("unroll") for (int i = 0; i < 8; i++) c2[i] = make_float2(0.f, 0.f);                            \
            cb2_tc_kstep(xt, v, wfrag + (((H) * CB2_TC_KSTEPS + 15) * 32 + lane_) * 2, c2);                         \
            _Pragma("unroll") for (int i = 0; i < 8; i++)                                                           \
                o2[i] = make_float2(__fadd_rn(o2[i].x, c2[i].x), __fadd_rn(o2[i].y, c2[i].y));                      \
        }                                                                                                           \
        _Pragma("unroll") for (int k = 0; k < 8; k++)                                                               \
            _Pragma("unroll") for (int c4 = 0; c4 < 4; c4++) {                                                      \
                if constexpr (!TC) {                                                                                \
                    const float4 w4 = *reinterpret_cast<const float4 *>(&P.root[8 * (H) + k][4 * c4]);              \
                    o2[2 * c4] = ffma2(make_float2(v[k], v[k]), make_float2(w4.x, w4.y), o2[2 * c4]);               \
                    o2[2 * c4 + 1] = ffma2(make_float2(v[k], v[k]), make_float2(w4.z, w4.w), o2[2 * c4 + 1]);       \
                }                                                                                                   \
                if constexpr (MODE_A) {                 /* the layer's skip branch Linear(x0) (conv.py:41-52) */    \
                    const float4 k4 = *reinterpret_cast<const float4 *>(&P.skip[8 * (H) + k][4 * c4]);              \
                    sk2[2 * c4] = ffma2(make_float2(v[k], v[k]), make_float2(k4.x, k4.y), sk2[2 * c4]);             \
                    sk2[2 * c4 + 1] = ffma2(make_float2(v[k], v[k]), make_float2(k4.z, k4.w), sk2[2 * c4 + 1]);     \
                }                                                                                                   \
            }                                                                                                       \
    } while (0)
                if (!sparse || wid_ == 0) {
                    if (half == 0)      CB2_ROOT(0);
                    else if (half == 1) CB2_ROOT(1);
                    else if constexpr (NCH > 2) CB2_ROOT(2);
                }
#undef CB2_ROOT
#define CB2_PASS(H, G)                                                                                               \
    do {                                                                                                            \
        if (staged) cb2_pass<true, H, G, THREADS, TC>(N, p, nn, xa, s_rows, s_wx, s_wy, s_wy4, s_ell, s_sp, nbr, off, P, wfrag, xt, p + d1, g.r, tix, o2); \
        else        cb2_pass<false, H, G, THREADS, TC>(N, p, nn, xa, s_rows, s_wx, s_wy, s_wy4, s_ell, s_sp, nbr, off, P, wfrag, xt, 0, g.r, tix, o2);     \
    } while (0)
#define CB2_HALF(H)                                                                                                  \
    do {                                                                                                            \
        if (!sparse) { CB2_PASS(H, 0); CB2_PASS(H, 1); CB2_PASS(H, 2); }                                            \
        else if (wid_ == 0) CB2_PASS(H, 0);                                                                         \
        else if (wid_ == 1) CB2_PASS(H, 1);                                                                         \
        else CB2_PASS(H, 2);                                                                                        \
    } while (0)
                if (half == 0)      CB2_HALF(0);
                else if (half == 1) CB2_HALF(1);
                else if constexpr (NCH > 2) CB2_HALF(2);
#undef CB2_HALF
#undef CB2_PASS
            }
        }
        if constexpr (TC) {
            if (__any_sync(0xffffffffu, active)) cb2_tc_unfrag(xt, o2);
        }
        if (sparse) {
            // add the partial sums of warps 1 and 2 (x-slots 1 and 2) to warp 0's: the staged rows are dead by now
            __syncthreads();
            float *s_part = s_rows;                                         // [2][32][16]
            if (active && wid_ >= 1) {
                float4 *dst = reinterpret_cast<float4 *>(s_part + ((size_t)(wid_ - 1) * 32 + lane_) * 16);
                dst[0] = make_float4(o2[0].x, o2[0].y, o2[1].x, o2[1].y);
                dst[1] = make_float4(o2[2].x, o2[2].y, o2[3].x, o2[3].y);
                dst[2] = make_float4(o2[4].x, o2[4].y, o2[5].x, o2[5].y);
                dst[3] = make_float4(o2[6].x, o2[6].y, o2[7].x, o2[7].y);
            }
            __syncthreads();
            if (active && wid_ == 0) {
#pragma unroll
                for (int w2 = 0; w2 < 2; w2++) {
                    const float4 *src = reinterpret_cast<const float4 *>(s_part + ((size_t)w2 * 32 + lane_) * 16);
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const float4 v = src[k];
                        o2[2 * k].x += v.x; o2[2 * k].y += v.y; o2[2 * k + 1].x += v.z; o2[2 * k + 1].y += v.w;
                    }
                }
            }
        }
        const bool owner = !sparse || wid_ == 0;                            // the thread that finishes this node
        if (!MODE_A && inrange && owner) { const uint32_t w0 = xyb[p]; const int t0 = ti[p].x; sx += w0 & 0xfff; sy += (w0 >> 12) & 0xfff; st += t0; tm = max(tm, t0); }
        if (!active || !owner) continue;
        float o[16];
#pragma unroll
        for (int c = 0; c < 8; c++) { o[2 * c] = o2[c].x; o[2 * c + 1] = o2[c].y; }
        if constexpr (MODE_A) {
            float sk[16];
#pragma unroll
            for (int c = 0; c < 8; c++) { sk[2 * c] = sk2[c].x; sk[2 * c + 1] = sk2[c].y; }
            const int sw = XA_SWZ(p);
            {
                // the (polarity, x, y) channels of the 19-channel conv were summed by the probe kernel (they need no
                // gather: dagr_l1_build with the event-channel weights, no BN / act) and wait in this node's xa row;
                // their part of the skip branch Linear(x0) is three FMAs per output here
                const float4 *pp = reinterpret_cast<const float4 *>(xa_out + (int64_t)p * 8);
                const float4 a0 = pp[sw], a1 = pp[sw ^ 1];
                pp = reinterpret_cast<const float4 *>(xa_out + (N + (int64_t)p) * 8);
                const float4 a2 = pp[sw], a3 = pp[sw ^ 1];
                const float part[16] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w, a3.x, a3.y, a3.z, a3.w};
                const uint32_t wxy = xyb[p];
                const float f0 = feat_s[p], f1 = __ldg(g.posx0 + (wxy & 0xfff)), f2 = __ldg(g.posy0 + ((wxy >> 12) & 0xfff));
#pragma unroll
                for (int c = 0; c < 16; c++) {
                    o[c] += part[c];
                    sk[c] = fmaf(f0, P.skip[16][c], sk[c]);
                    sk[c] = fmaf(f1, P.skip[17][c], sk[c]);
                    sk[c] = fmaf(f2, P.skip[18][c], sk[c]);
                }
            }
#pragma unroll
            for (int c = 0; c < 16; c++) {
                const float r = fmaf(o[c], P.scale[c], P.shift[c]);
                o[c] = relu ? fmaxf(r, 0.f) : r;
                sk[c] = fmaf(sk[c], P.sscale[c], P.sshift[c]);
            }
            float4 *dst = reinterpret_cast<float4 *>(xa_out + (int64_t)p * 8);
            dst[sw] = make_float4(o[0], o[1], o[2], o[3]);
            dst[sw ^ 1] = make_float4(o[4], o[5], o[6], o[7]);
            dst = reinterpret_cast<float4 *>(xa_out + (N + (int64_t)p) * 8);
            dst[sw] = make_float4(o[8], o[9], o[10], o[11]);
            dst[sw ^ 1] = make_float4(o[12], o[13], o[14], o[15]);
            float4 *sd = reinterpret_cast<float4 *>(skip_out + (int64_t)p * 16);
            sd[0] = make_float4(sk[0], sk[1], sk[2], sk[3]);
            sd[1] = make_float4(sk[4], sk[5], sk[6], sk[7]);
            sd[2] = make_float4(sk[8], sk[9], sk[10], sk[11]);
            sd[3] = make_float4(sk[12], sk[13], sk[14], sk[15]);
            continue;
        }
        const uint32_t wxy = xyb[p];
        const int x = wxy & 0xfff, y = (wxy >> 12) & 0xfff;
        float skv[16];
        if (skip_pre != nullptr) {
            const float4 *sp = reinterpret_cast<const float4 *>(skip_pre + (int64_t)p * 16);
            const float4 a = sp[0], b4 = sp[1], c4 = sp[2], d4 = sp[3];
            skv[0] = a.x; skv[1] = a.y; skv[2] = a.z; skv[3] = a.w; skv[4] = b4.x; skv[5] = b4.y; skv[6] = b4.z; skv[7] = b4.w;
            skv[8] = c4.x; skv[9] = c4.y; skv[10] = c4.z; skv[11] = c4.w; skv[12] = d4.x; skv[13] = d4.y; skv[14] = d4.z; skv[15] = d4.w;
        } else {
            const float f0 = feat_s[p], f1 = __ldg(g.posx0 + x), f2 = __ldg(g.posy0 + y);
#pragma unroll
            for (int c = 0; c < 16; c++) {
                float sk = f0 * P.skip[0][c];
                sk = fmaf(f1, P.skip[1][c], sk);
                sk = fmaf(f2, P.skip[2][c], sk);
                skv[c] = fmaf(sk, P.sscale[c], P.sshift[c]);
            }
        }
#pragma unroll
        for (int c = 0; c < 16; c++) {
            float r = fmaf(o[c], P.scale[c], P.shift[c]) + skv[c];
            r = relu ? fmaxf(r, 0.f) : r;
            o[c] = r;
        }
#pragma unroll
        for (int c = 0; c < 16; c++) m[c] = pool_mean ? m[c] + o[c] : fmaxf(m[c], o[c]);
        if (x1 != nullptr) {
            float4 *dst = reinterpret_cast<float4 *>(x1 + (int64_t)p * 16);
            dst[0] = make_float4(o[0], o[1], o[2], o[3]);
            dst[1] = make_float4(o[4], o[5], o[6], o[7]);
            dst[2] = make_float4(o[8], o[9], o[10], o[11]);
            dst[3] = make_float4(o[12], o[13], o[14], o[15]);
        }
    }
    if (MODE_A) return;
    // ---- pool1: per-voxel max / mean position (pooling.py:66-86) -------------------------------------
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
#pragma unroll
        for (int c = 0; c < 16; c++) {
            const float o2 = __shfl_xor_sync(0xffffffffu, m[c], d);
            m[c] = pool_mean ? m[c] + o2 : fmaxf(m[c], o2);
        }
        sx += __shfl_xor_sync(0xffffffffu, sx, d);
        sy += __shfl_xor_sync(0xffffffffu, sy, d);
        st += __shfl_xor_sync(0xffffffffu, st, d);
        tm = max(tm, __shfl_xor_sync(0xffffffffu, tm, d));
    }
    if (lane == 0) {
#pragma unroll
        for (int c = 0; c < 16; c++) s_red[wid][c] = m[c];
        s_sum[wid][0] = sx; s_sum[wid][1] = sy; s_sum[wid][2] = st; s_tm[wid] = tm;
    }
    __syncthreads();
    const int nw = blockDim.x >> 5;
    if (threadIdx.x < 16) {
        float v = s_red[0][threadIdx.x];
        for (int w2 = 1; w2 < nw; w2++) v = pool_mean ? v + s_red[w2][threadIdx.x] : fmaxf(v, s_red[w2][threadIdx.x]);
        if (pool_mean) v = __fdiv_rn(v, (float)nown);                   // scatter_mean: sum / count
        if (persist != nullptr) {                                        // running per-voxel max of the stream
            if (min_idx > 0) v = fmaxf(v, persist[(int64_t)cell * 16 + threadIdx.x]);
            persist[(int64_t)cell * 16 + threadIdx.x] = v;
        }
        xg[(int64_t)cell * ldx + threadIdx.x] = v;
    }
    if (threadIdx.x == 32) {
        long long ax = 0, ay = 0, at = 0; int tmx = -2147483647;
        for (int w2 = 0; w2 < nw; w2++) { ax += s_sum[w2][0]; ay += s_sum[w2][1]; at += s_sum[w2][2]; tmx = max(tmx, s_tm[w2]); }
        const float mx = (float)((double)ax / ((double)nown * (double)g.W));
        const float my = (float)((double)ay / ((double)nown * (double)g.H));
        cnt[cell] = nown;
        pxy[2 * cell] = cb2_round_to_pixel(mx, g.W);
        pxy[2 * cell + 1] = cb2_round_to_pixel(my, g.H);
        tmean[cell] = (float)((double)at / ((double)nown * (double)g.T));
        tmax[cell] = __fdiv_rn((float)tmx, (float)g.T);
    }
}


template <class PT, int NCH, bool MODE_A, bool POOL_MEAN, bool PLAIN, bool TC>
__global__ void __launch_bounds__(CB2_THREADS, MODE_A ? 3 : 4)       // (3 CTAs / 128 registers, no spills: slower)
k_l1_conv_b2(const dagr_geom_t g, int64_t N, const int32_t *__restrict__ start, const uint32_t *__restrict__ xyb,
             const int2 *__restrict__ ti, const float *__restrict__ feat_s, const float *__restrict__ xa,
             const int32_t *__restrict__ nbr, const uint16_t *__restrict__ off,
             const __grid_constant__ PT P, const float4 *__restrict__ wfrag, const float *__restrict__ skip_pre, const int min_idx,
             float *__restrict__ persist, float *__restrict__ x1, int32_t *__restrict__ cnt, int32_t *__restrict__ pxy,
             float *__restrict__ tmean, float *__restrict__ tmax, float *__restrict__ xg, int ldx,
             float *__restrict__ xa_out, float *__restrict__ skip_out, int32_t *__restrict__ wl_hdr, int32_t *__restrict__ wl_ids,
             const int defer)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(16) CB2Shared<CB2_THREADS> S;
    if (threadIdx.x == 0) mbar_init(&S.bar, 1);                         // made visible by the routine's first __syncthreads
    uint32_t parity = 0;
    cb2_voxel<PT, NCH, MODE_A, CB2_CAP, CB2_THREADS, POOL_MEAN, PLAIN, TC>(g, N, start, xyb, ti, feat_s, xa, nbr, off, P, wfrag, skip_pre, min_idx,
                                                      persist, x1, cnt, pxy, tmean, tmax, xg, ldx, xa_out, skip_out, (int)blockIdx.x,
                                                      smem_raw, S, parity, wl_hdr, wl_ids, defer);
}

// dense voxels: persistent CTAs (one per SM) pop voxel ids from the work list the regular kernel filled
template <class PT, int NCH, bool MODE_A, bool POOL_MEAN, bool PLAIN, bool TC>
__global__ void __launch_bounds__(CB2_THREADS_BIG, 1)
k_l1_conv_b2_dense(const dagr_geom_t g, int64_t N, const int32_t *__restrict__ start, const uint32_t *__restrict__ xyb,
                   const int2 *__restrict__ ti, const float *__restrict__ feat_s, const float *__restrict__ xa,
                   const int32_t *__restrict__ nbr, const uint16_t *__restrict__ off,
                   const __grid_constant__ PT P, const float4 *__restrict__ wfrag, const float *__restrict__ skip_pre, const int min_idx,
                   float *__restrict__ persist, float *__restrict__ x1, int32_t *__restrict__ cnt, int32_t *__restrict__ pxy,
                   float *__restrict__ tmean, float *__restrict__ tmax, float *__restrict__ xg, int ldx,
                   float *__restrict__ xa_out, float *__restrict__ skip_out, int32_t *__restrict__ wl_hdr, const int32_t *__restrict__ wl_ids)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(16) CB2Shared<CB2_THREADS_BIG> S;
    __shared__ int s_next;
    if (threadIdx.x == 0) mbar_init(&S.bar, 1);
    uint32_t parity = 0;                                                // the barrier's phase carries over from voxel to voxel
    const int count = wl_hdr[0];
    for (;;) {
        __syncthreads();                                                // everyone is done with the previous voxel
        if (threadIdx.x == 0) s_next = atomicAdd(&wl_hdr[1], 1);
        __syncthreads();
        const int i = s_next;
        if (i >= count) break;
        cb2_voxel<PT, NCH, MODE_A, CB2_CAP_BIG, CB2_THREADS_BIG, POOL_MEAN, PLAIN, TC>(g, N, start, xyb, ti, feat_s, xa, nbr, off, P, wfrag, skip_pre,
                                                                  min_idx, persist, x1, cnt, pxy, tmean, tmax, xg, ldx, xa_out, skip_out,
                                                                  wl_ids[i], smem_raw, S, parity, nullptr, nullptr, 0);
    }
}

static size_t cb2_smem_bytes(const dagr_geom_t *g, int cap, int threads)
{
    return (size_t)cap * 32 + 96 * 16 + (size_t)DAGR_ELL * threads * 4 + (size_t)g->ncell * 2 + 32;
}

template <class PT, int NCH, bool MODE_A, bool TC, bool POOL_MEAN = false, bool PLAIN = false>
static int cb2_launch(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int2 *ti, const float *feat_s,
                      const float *xa, const int32_t *nbr, const uint16_t *off, const PT *p_host, const float4 *wfrag, const float *skip_pre,
                      int min_idx, float *persist, float *x1, int32_t *cnt, int32_t *pxy, float *tmean, float *tmax, float *xg, int ldx,
                      float *xa_out, float *skip_out, int32_t *wl_hdr, int32_t *wl_ids, int defer, cudaStream_t st)
{
    const int cells = g->B * g->ny1 * g->nx1;
    const size_t smem = cb2_smem_bytes(g, CB2_CAP, CB2_THREADS);
    auto kern = k_l1_conv_b2<PT, NCH, MODE_A, POOL_MEAN, PLAIN, TC>;
    DAGR_CUDA(dagr_allow_smem(kern, smem, true));
    kern<<<cells, CB2_THREADS, smem, st>>>(*g, N, start, xyb, ti, feat_s, xa, nbr, off, *p_host, wfrag, skip_pre, min_idx, persist, x1, cnt,
                                           pxy, tmean, tmax, xg, ldx, xa_out, skip_out, wl_hdr, wl_ids,
                                           (wl_hdr != nullptr && wl_ids != nullptr && defer) ? 1 : 0);
    DAGR_CHECK_LAUNCH();
    if (wl_hdr != nullptr && wl_ids != nullptr && defer) {
        static int n_sm = 0;
        if (n_sm == 0) {
            int dev = 0;
            DAGR_CUDA(cudaGetDevice(&dev));
            DAGR_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        }
        const size_t smem_big = cb2_smem_bytes(g, CB2_CAP_BIG, CB2_THREADS_BIG);
        auto kd = k_l1_conv_b2_dense<PT, NCH, MODE_A, POOL_MEAN, PLAIN, TC>;
        DAGR_CUDA(dagr_allow_smem(kd, smem_big));
        kd<<<n_sm, CB2_THREADS_BIG, smem_big, st>>>(*g, N, start, xyb, ti, feat_s, xa, nbr, off, *p_host, wfrag, skip_pre, min_idx, persist,
                                                    x1, cnt, pxy, tmean, tmax, xg, ldx, xa_out, skip_out, wl_hdr, wl_ids);
        DAGR_CHECK_LAUNCH();
    }
    return DAGR_OK;
}

template <bool TC>
static int conv_b_pool_voxel(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                             const float *feat_s, const float *xa, const int32_t *nbr, const uint16_t *off, const dagr_l1b_params_t *p_host,
                             const float4 *wfrag, const float *skip_pre, int min_idx, float *persist, float *x1, int32_t *cnt,
                             int32_t *pxy, float *tmean, float *tmax, float *xg, int ldx, int32_t *wl_hdr, int32_t *wl_ids, int defer,
                             cudaStream_t st)
{
    DAGR_CHECK_ARG(g && p_host, "null argument");
    DAGR_CHECK_ARG(g->r <= 15, "radius must be <= 15 px (offsets are packed in 5 bits)");
    DAGR_CHECK_ARG(!(p_host->pool_mean && persist), "the running per-voxel aggregate of the event stream is a max (max_pool.py:59-62)");
    if (p_host->pool_mean)
        return cb2_launch<dagr_l1b_params_t, 2, false, TC, true>(g, N, start, xyb, (const int2 *)ti, feat_s, xa, nbr, off, p_host, wfrag,
                                                                 skip_pre, min_idx, persist, x1, cnt, pxy, tmean, tmax, xg, ldx, nullptr,
                                                                 nullptr, wl_hdr, wl_ids, defer, st);
    if (min_idx <= 0 && persist == nullptr && x1 == nullptr && skip_pre == nullptr && p_host->relu)
        return cb2_launch<dagr_l1b_params_t, 2, false, TC, false, true>(g, N, start, xyb, (const int2 *)ti, feat_s, xa, nbr, off, p_host, wfrag,
                                                                        nullptr, 0, nullptr, nullptr, cnt, pxy, tmean, tmax, xg, ldx, nullptr,
                                                                        nullptr, wl_hdr, wl_ids, defer, st);
    return cb2_launch<dagr_l1b_params_t, 2, false, TC>(g, N, start, xyb, (const int2 *)ti, feat_s, xa, nbr, off, p_host, wfrag, skip_pre,
                                                       min_idx, persist, x1, cnt, pxy, tmean, tmax, xg, ldx, nullptr, nullptr, wl_hdr, wl_ids,
                                                       defer, st);
}

extern "C" int dagr_l1_conv_b_pool_voxel(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                                         const int32_t *ti, const float *feat_s, const float *xa, const int32_t *nbr,
                                         const uint16_t *off, const float *tab, const dagr_l1b_params_t *p_host,
                                         const float *skip_pre, int min_idx, float *persist, float *x1, int32_t *cnt,
                                         int32_t *pxy, float *tmean, float *tmax, float *xg, int ldx, int32_t *wl_hdr, int32_t *wl_ids,
                                         int defer, void *stream)
{
    (void)tab;
    return conv_b_pool_voxel<false>(g, N, start, xyb, ti, feat_s, xa, nbr, off, p_host, nullptr, skip_pre, min_idx, persist, x1, cnt, pxy,
                                    tmean, tmax, xg, ldx, wl_hdr, wl_ids, defer, (cudaStream_t)stream);
}

extern "C" int dagr_l1_conv_b_pool_voxel_tc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                                            const int32_t *ti, const float *feat_s, const float *xa, const int32_t *nbr,
                                            const uint16_t *off, const dagr_l1b_params_t *p_host, const float *wfrag,
                                            const float *skip_pre, int min_idx, float *persist, float *x1, int32_t *cnt,
                                            int32_t *pxy, float *tmean, float *tmax, float *xg, int ldx, int32_t *wl_hdr, int32_t *wl_ids,
                                            int defer, void *stream)
{
    DAGR_CHECK_ARG(wfrag, "null weight fragments (dagr_l1_tc_weights)");
    return conv_b_pool_voxel<CB2_TC != 0>(g, N, start, xyb, ti, feat_s, xa, nbr, off, p_host, (const float4 *)wfrag, skip_pre, min_idx,
                                          persist, x1, cnt, pxy, tmean, tmax, xg, ldx, wl_hdr, wl_ids, defer, (cudaStream_t)stream);
}

// image fusion: the 16 image channels of conv_block1.conv_block1 (x0 chunk-major [2][N][8], chunks swizzled like xa) on top
// of the event-channel sums the probe kernel left in xa
template <bool TC>
static int conv_a_image(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s, const float *x0,
                        const int32_t *nbr, const uint16_t *off, const dagr_l1img_params_t *p_host, const float4 *wfrag, float *xa,
                        float *skipv, int32_t *wl_hdr, int32_t *wl_ids, int defer, cudaStream_t st)
{
    DAGR_CHECK_ARG(g && p_host && xyb && feat_s, "null argument");
    if (N <= 0) return DAGR_OK;
    DAGR_CHECK_ARG(g->r <= 15, "radius must be <= 15 px (offsets are packed in 5 bits)");
    return cb2_launch<dagr_l1img_params_t, 2, true, TC>(g, N, start, xyb, nullptr, feat_s, x0, nbr, off, p_host, wfrag, nullptr, 0, nullptr,
                                                        nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, xa, skipv, wl_hdr, wl_ids,
                                                        defer, st);
}

extern "C" int dagr_l1_conv_a_image(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s,
                                    const float *x0, const int32_t *nbr,
                                    const uint16_t *off, const dagr_l1img_params_t *p_host, float *xa, float *skipv,
                                    int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream)
{
    return conv_a_image<false>(g, N, start, xyb, feat_s, x0, nbr, off, p_host, nullptr, xa, skipv, wl_hdr, wl_ids, defer, (cudaStream_t)stream);
}

extern "C" int dagr_l1_conv_a_image_tc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s,
                                       const float *x0, const int32_t *nbr, const uint16_t *off, const dagr_l1img_params_t *p_host,
                                       const float *wfrag, float *xa, float *skipv, int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream)
{
    DAGR_CHECK_ARG(wfrag, "null weight fragments (dagr_l1_tc_weights)");
    return conv_a_image<CB2_TC != 0>(g, N, start, xyb, feat_s, x0, nbr, off, p_host, (const float4 *)wfrag, xa, skipv, wl_hdr, wl_ids, defer,
                                     (cudaStream_t)stream);
}

// incremental stream step of the same instances: only nodes with arrival index ti[p].y >= min_idx are convolved, their xa rows
// (the probe's event-channel sums) finished and their skipv rows written.  The rows of older nodes hold final activations
// gathered from arrival storage and are not touched.  min_idx == 0 takes every node: the bits of dagr_l1_conv_a_image_tc.
extern "C" int dagr_l1_conv_a_image_inc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                                        const float *feat_s, const float *x0, const int32_t *nbr, const uint16_t *off,
                                        const dagr_l1img_params_t *p_host, const float *wfrag, int min_idx, float *xa, float *skipv,
                                        int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream)
{
    DAGR_CHECK_ARG(g && start && xyb && ti && feat_s && x0 && nbr && off && p_host && wfrag && xa && skipv,
                   "null argument (only wl_hdr / wl_ids may be NULL)");
    DAGR_CHECK_ARG(min_idx >= 0, "min_idx must be >= 0");
    DAGR_CHECK_ARG(N >= 0 && N < (1ll << 31), "N out of range");
    if (N == 0) return DAGR_OK;
    DAGR_CHECK_ARG(g->r <= 15, "radius must be <= 15 px (offsets are packed in 5 bits)");
    return cb2_launch<dagr_l1img_params_t, 2, true, CB2_TC != 0>(g, N, start, xyb, (const int2 *)ti, feat_s, x0, nbr, off, p_host,
                                                                  (const float4 *)wfrag, nullptr, min_idx, nullptr, nullptr, nullptr,
                                                                  nullptr, nullptr, nullptr, nullptr, 0, xa, skipv, wl_hdr, wl_ids, defer,
                                                                  (cudaStream_t)stream);
}

// host-side packing of the weight fragments the tensor-core instances read (layout: see cb2_tc_kstep)
extern "C" int dagr_l1_tc_weights(const float *w_host, const float *root_host, int cin, float *wfrag_host)
{
    DAGR_CHECK_ARG(w_host && root_host && wfrag_host, "null argument");
    DAGR_CHECK_ARG(cin >= 16, "the tensor-core instances take input channels 0..15");
    for (int half = 0; half < 2; half++)
        for (int s = 0; s < CB2_TC_KSTEPS; s++)
            for (int lane = 0; lane < 32; lane++)
                for (int nt = 0; nt < 2; nt++) {
                    const int g = lane >> 2, t = lane & 3, n = 8 * nt + g;
                    const float *W = s < DAGR_KU ? w_host + (size_t)s * cin * 16 : root_host;
                    const float x0 = W[(8 * half + t) * 16 + n], x1 = W[(8 * half + t + 4) * 16 + n];
                    const float h0 = tf32_rna_host(x0), h1 = tf32_rna_host(x1);
                    float *o = wfrag_host + ((((size_t)half * CB2_TC_KSTEPS + s) * 32 + lane) * 2 + nt) * 4;
                    o[0] = h0; o[1] = h1; o[2] = x0 - h0; o[3] = x1 - h1;
                }
    return DAGR_OK;
}


// ------------------------------------------------------------------------------------------------
// streaming support: node rows live in arrival order between steps (the cell-major order changes whenever
// events are appended); gather old rows into the new sorted order / scatter freshly computed rows back.
// xa_sorted is half-major [2][N][8]; xa_arrival is row-major [cap][16].
// ------------------------------------------------------------------------------------------------
__global__ void k_xa_permute(int64_t N, const int32_t *__restrict__ perm, int n_old, float *__restrict__ xa_sorted,
                             float *__restrict__ xa_arrival, int scatter)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t p = t >> 2;
    const int q = (int)(t & 3);
    if (p >= N) return;
    const int i = perm[p];
    float4 *srt = reinterpret_cast<float4 *>(xa_sorted + ((int64_t)(q >> 1) * N + p) * 8) + ((q & 1) ^ XA_SWZ(p));
    float4 *arr = reinterpret_cast<float4 *>(xa_arrival + (int64_t)i * 16) + q;
    if (scatter) { if (i >= n_old) *arr = *srt; }
    else         { if (i < n_old) *srt = *arr; }
}

extern "C" int dagr_xa_permute(int64_t N, const int32_t *perm, int n_old, float *xa_sorted, float *xa_arrival, int scatter, void *stream)
{
    if (N <= 0) return DAGR_OK;
    k_xa_permute<<<dagr_div_up(4 * N, 256), 256, 0, (cudaStream_t)stream>>>(N, perm, n_old, xa_sorted, xa_arrival, scatter);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}
