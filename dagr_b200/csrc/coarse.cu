// coarse.cu -- everything after the event level: voxel-grid pooling, SplineConv on voxel grids,
// dense projection, decode and NMS.  sm_90a.
//
// After pool1 the graph has at most B*56*40 nodes and, because the event radius (r px) is smaller
// than a pool1 voxel, every coarse edge joins 8-neighbouring voxels.  The coarse levels are therefore
// stored as DENSE voxel grids [B, ny, nx] (valid flag, rounded pixel position, features, 8-bit
// in-edge mask) instead of the reference's compacted node/edge lists (pooling.py:51-97).  The
// reference's consecutive node ids / sorted unique edge lists are recovered from the grids on demand
// (dagr_b200/export.py) for parity checks.
#include "common.cuh"

// ------------------------------------------------------------------------------------------------
// pool1 finalize: one warp per voxel
// ------------------------------------------------------------------------------------------------
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

__device__ __forceinline__ int round_to_pixel(float mean, int size)
{
    // floor((pos + 1e-5) / (1/size))   (pooling.py:47-49), wh_inv = fl(1/size)
    const float inv = __frcp_rn((float)size);
    const float q = div_floor_f32(__fadd_rn(mean, 1e-5f), inv);
    const int k = (int)q;
    return min(max(k, 0), size - 1);
}

__global__ void __launch_bounds__(128)
k_pool1_finalize(const dagr_geom_t g, const int32_t *__restrict__ start, const uint32_t *__restrict__ xyb,
                 const int2 *__restrict__ ti, const uint32_t *__restrict__ poolmax, int C,
                 int32_t *__restrict__ cnt, int32_t *__restrict__ pxy, float *__restrict__ tmean,
                 float *__restrict__ tmax, float *__restrict__ x)
{
    const int cells = g.B * g.ny1 * g.nx1;
    const int cell = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (cell >= cells) return;
    const int s = start[(int64_t)cell * g.CP], e = start[(int64_t)(cell + 1) * g.CP];
    long long sx = 0, sy = 0, st = 0;
    int tm = -2147483647;
    for (int p = s + lane; p < e; p += 32) {
        const uint32_t w = xyb[p];
        sx += w & 0xfff; sy += (w >> 12) & 0xfff;
        const int t = ti[p].x;
        st += t; tm = max(tm, t);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        sx += __shfl_xor_sync(0xffffffffu, sx, d);
        sy += __shfl_xor_sync(0xffffffffu, sy, d);
        st += __shfl_xor_sync(0xffffffffu, st, d);
        tm = max(tm, __shfl_xor_sync(0xffffffffu, tm, d));
    }
    const int n = e - s;
    if (lane == 0) {
        cnt[cell] = n;
        if (n > 0) {
            const float mx = (float)((double)sx / ((double)n * (double)g.W));
            const float my = (float)((double)sy / ((double)n * (double)g.H));
            pxy[2 * cell] = round_to_pixel(mx, g.W);
            pxy[2 * cell + 1] = round_to_pixel(my, g.H);
            tmean[cell] = (float)((double)st / ((double)n * (double)g.T));
            tmax[cell] = __fdiv_rn((float)tm, (float)g.T);
        } else {
            pxy[2 * cell] = 0; pxy[2 * cell + 1] = 0; tmean[cell] = 0.f; tmax[cell] = 0.f;
        }
    }
    for (int c = lane; c < C; c += 32)
        x[(int64_t)cell * C + c] = n > 0 ? dec_ordered(poolmax[(int64_t)cell * C + c]) : 0.f;
}

extern "C" int dagr_pool1_finalize(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                                   const int32_t *ti, const uint32_t *poolmax, int C, int32_t *cnt, int32_t *pxy,
                                   float *tmean, float *tmax, float *x, void *stream)
{
    (void)N;
    const int cells = g->B * g->ny1 * g->nx1;
    k_pool1_finalize<<<dagr_div_up(cells, 4), 128, 0, (cudaStream_t)stream>>>(*g, start, xyb, (const int2 *)ti, poolmax, C,
                                                                            cnt, pxy, tmean, tmax, x);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// cat(x, pos[:, :2])
// ------------------------------------------------------------------------------------------------
__global__ void k_cat_pos(const dagr_grid_t gr, const int32_t *__restrict__ cnt, const int32_t *__restrict__ pxy,
                          const float *__restrict__ x, int Cx, float *__restrict__ xin, int64_t total)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int Ci = Cx + 2;
    const int64_t cell = i / Ci;
    const int c = (int)(i % Ci);
    float v = 0.f;
    if (cnt[cell] > 0) {
        if (c < Cx) v = x[cell * Cx + c];
        else if (c == Cx) v = gr.posxr[pxy[2 * cell]];
        else v = gr.posyr[pxy[2 * cell + 1]];
    }
    xin[i] = v;
}

extern "C" int dagr_grid_cat_pos(const dagr_grid_t *gr, const int32_t *cnt, const int32_t *pxy, const float *x, int Cx,
                                 float *xin, void *stream)
{
    const int64_t total = (int64_t)gr->B * gr->ny * gr->nx * (Cx + 2);
    k_cat_pos<<<dagr_div_up(total, 256), 256, 0, (cudaStream_t)stream>>>(*gr, cnt, pxy, x, Cx, xin, total);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// SplineConv on a voxel grid: one warp per destination voxel (v1: direct slot form)
// ------------------------------------------------------------------------------------------------
#define GC_WARPS 4
#define GC_SLOTS 25

__global__ void __launch_bounds__(GC_WARPS * 32)
k_grid_conv(const dagr_grid_t gr, const int32_t *__restrict__ cnt, const int32_t *__restrict__ pxy,
            const uint32_t *__restrict__ mask, const float *__restrict__ xin, int ldin, int Cin, int Cout,
            const float *__restrict__ weight, const float *__restrict__ rootT, const float *__restrict__ bias,
            const float *__restrict__ scale, const float *__restrict__ shift, const float *__restrict__ skip,
            int relu, float den_x, float den_y, float *__restrict__ out)
{
    extern __shared__ __align__(16) float smem_f[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float *A = smem_f + (size_t)warp * GC_SLOTS * Cin;          // [25][Cin]
    const int cells = gr.B * gr.ny * gr.nx;
    const int cell = blockIdx.x * GC_WARPS + warp;
    if (cell >= cells) return;
    if (cnt[cell] <= 0) {
        for (int o = lane; o < Cout; o += 32) out[(int64_t)cell * Cout + o] = 0.f;
        return;
    }
    const int per = gr.ny * gr.nx;
    const int b = cell / per, rem = cell % per, cy = rem / gr.nx, cx = rem % gr.nx;
    const int px = pxy[2 * cell], py = pxy[2 * cell + 1];
    const uint32_t m = mask[cell];
    uint32_t used = 0;

    for (int i = lane; i < GC_SLOTS * Cin; i += 32) A[i] = 0.f;
    __syncwarp();
    for (int bit = 0; bit < 9; bit++) {
        if (!((m >> bit) & 1u) || bit == 4) continue;
        const int dcx = bit % 3 - 1, dcy = bit / 3 - 1;
        const int sx = cx + dcx, sy = cy + dcy;
        if (sx < 0 || sy < 0 || sx >= gr.nx || sy >= gr.ny) continue;
        const int src = b * per + sy * gr.nx + sx;
        if (cnt[src] <= 0) continue;
        const int dx = pxy[2 * src] - px, dy = pxy[2 * src + 1] - py;
        // attr = d / (2*M*size) + 0.5 exactly as init_lut evaluates it (spline_conv.py:28-29)
        const float ax = __fadd_rn(__fdiv_rn((float)dx, den_x), 0.5f);
        const float ay = __fadd_rn(__fdiv_rn((float)dy, den_y), 0.5f);
        float w[4]; int slot[4];
        spline_basis2(ax, ay, 5, w, slot);
        const float *xs = xin + (int64_t)src * ldin;
        for (int ci = lane; ci < Cin; ci += 32) {
            const float v = xs[ci];
#pragma unroll
            for (int s = 0; s < 4; s++) A[slot[s] * Cin + ci] = fmaf(w[s], v, A[slot[s] * Cin + ci]);
        }
#pragma unroll
        for (int s = 0; s < 4; s++) if (w[s] != 0.f) used |= 1u << slot[s];
    }
    __syncwarp();
    const float *xd = xin + (int64_t)cell * ldin;
    for (int o = lane; o < Cout; o += 32) {
        float acc = 0.f;
        uint32_t u = used;
        while (u) {
            const int k = __ffs(u) - 1; u &= u - 1;
            const float *wk = weight + (int64_t)k * Cin * Cout + o;
            const float *ak = A + k * Cin;
            for (int ci = 0; ci < Cin; ci++) acc = fmaf(ak[ci], __ldg(wk + (int64_t)ci * Cout), acc);
        }
        for (int ci = 0; ci < Cin; ci++) acc = fmaf(xd[ci], __ldg(rootT + (int64_t)ci * Cout + o), acc);
        if (bias) acc += bias[o];
        if (scale) acc = fmaf(acc, scale[o], shift[o]);
        if (skip) acc += skip[(int64_t)cell * Cout + o];
        if (relu) acc = fmaxf(acc, 0.f);
        out[(int64_t)cell * Cout + o] = acc;
    }
}

// ------------------------------------------------------------------------------------------------
// v2: split-K SplineConv on a voxel grid.  One CTA handles CPB consecutive voxels with 8 warps:
//   phase 1  A[k][c][j] = sum_{in-edges e of voxel j} b_k(e) * x[src_e][c]   (k < 25), A[25] = x[j] (root)
//            built once in shared memory (each thread owns (voxel, channel) pairs: no races);
//   phase 2  warp w accumulates the slots k = w, w+8, ... : lanes run over output channels (coalesced
//            weight rows from L2), every weight is reused for all CPB voxels (A read as float4 broadcasts);
//   phase 3  the 8 partial sums meet in shared memory; bias, folded BN, residual and relu in the epilogue.
// The serial depth per lane drops from 25*Cin to ~3.3*Cin and each weight is fetched once per CPB voxels.
// ------------------------------------------------------------------------------------------------
#define SK_WARPS 8
#define SK_SLOTS 26

template <int CPB>
__global__ void __launch_bounds__(SK_WARPS * 32)
k_grid_conv_sk(const dagr_grid_t gr, const int32_t *__restrict__ cnt, const int32_t *__restrict__ pxy,
               const uint32_t *__restrict__ mask, const float *__restrict__ xin, int ldin, int Cin, int Cout,
               const float *__restrict__ weight, const float *__restrict__ rootT, const float *__restrict__ bias,
               const float *__restrict__ scale, const float *__restrict__ shift, const float *__restrict__ skip,
               int relu, float den_x, float den_y, float *__restrict__ out)
{
    extern __shared__ __align__(16) float smem_f[];
    float *A = smem_f;                                         // [26][Cin][CPB]
    // [SK_WARPS][CPB][Cout]; aliases A when there is a single 64-wide output tile (A is dead after phase 2)
    float *part = (Cout <= 64) ? A : A + (size_t)SK_SLOTS * Cin * CPB;
    // edge tables with the voxel index innermost: phase 1 runs with the voxel index fastest across lanes
    __shared__ int s_src[8][CPB];
    __shared__ float s_w[8][4][CPB];
    __shared__ unsigned char s_slot[8][4][CPB];
    __shared__ int s_ne[CPB];
    __shared__ unsigned int s_used;
    const int cells = gr.B * gr.ny * gr.nx;
    const int cell0 = blockIdx.x * CPB;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = gr.ny * gr.nx;

    if (tid == 0) s_used = 0;
    for (int i = tid; i < SK_SLOTS * Cin * CPB; i += blockDim.x) A[i] = 0.f;
    __syncthreads();
    // ---- edge tables: one thread per (voxel, neighbour bit) ---------------------------------------------
    if (tid < CPB * 9) {
        const int j = tid / 9, bit = tid % 9;
        const int cell = cell0 + j;
        if (bit == 4) {
            // slot bookkeeping done by the other lanes; this lane counts the edges afterwards
        } else if (cell < cells && cnt[cell] > 0 && ((mask[cell] >> bit) & 1u)) {
            const int b = cell / per, rem = cell % per, cy = rem / gr.nx, cx = rem % gr.nx;
            const int sx = cx + bit % 3 - 1, sy = cy + bit / 3 - 1;
            if (sx >= 0 && sy >= 0 && sx < gr.nx && sy < gr.ny) {
                const int src = b * per + sy * gr.nx + sx;
                if (cnt[src] > 0) {
                    const int dx = pxy[2 * src] - pxy[2 * cell], dy = pxy[2 * src + 1] - pxy[2 * cell + 1];
                    const float ax = __fadd_rn(__fdiv_rn((float)dx, den_x), 0.5f);
                    const float ay = __fadd_rn(__fdiv_rn((float)dy, den_y), 0.5f);
                    float w[4]; int slot[4];
                    spline_basis2(ax, ay, 5, w, slot);
                    const int e = bit < 4 ? bit : bit - 1;              // dense edge index 0..7
                    s_src[e][j] = src;
                    unsigned int used = 0;
#pragma unroll
                    for (int q = 0; q < 4; q++) { s_w[e][q][j] = w[q]; s_slot[e][q][j] = (unsigned char)slot[q]; if (w[q] != 0.f) used |= 1u << slot[q]; }
                    atomicOr(&s_used, used);
                    goto table_done;
                }
            }
            { const int e = bit < 4 ? bit : bit - 1; s_src[e][j] = -1; }
        } else {
            const int e = bit < 4 ? bit : bit - 1;
            if (bit != 4) s_src[e][j] = -1;
        }
    }
table_done:
    __syncthreads();
    // ---- phase 1: A[k][c][j] --------------------------------------------------------------------------------
    // the voxel index j runs fastest across the lanes: the read-modify-writes of A then touch CPB consecutive floats per
    // channel (conflict free for any mix of slots, since Cin*CPB is a multiple of 32 banks); with the channel fastest every
    // access of a warp fell on two banks (stride CPB floats: 16-way conflicts at CPB = 16).  The source rows sit in L2 / L1.
    for (int i = tid; i < CPB * Cin; i += blockDim.x) {
        const int j = i % CPB, c = i / CPB;
        const int cell = cell0 + j;
        if (cell >= cells || cnt[cell] <= 0) continue;
        A[((size_t)25 * Cin + c) * CPB + j] = xin[(int64_t)cell * ldin + c];          // root "slot"
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; e++) {                                                 // all gathers in flight before the updates
            const int src = s_src[e][j];
            v[e] = (src >= 0) ? xin[(int64_t)src * ldin + c] : 0.f;
        }
#pragma unroll
        for (int e = 0; e < 8; e++) {
            if (s_src[e][j] < 0) continue;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                float *a = A + ((size_t)s_slot[e][q][j] * Cin + c) * CPB + j;
                *a = fmaf(s_w[e][q][j], v[e], *a);
            }
        }
    }
    __syncthreads();
    // ---- phase 2: split-K over slots ---------------------------------------------------------------------------
    const unsigned int used = s_used | (1u << 25);
    for (int o0 = 0; o0 < Cout; o0 += 64) {
        float acc[2][CPB];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int j = 0; j < CPB; j++) acc[h][j] = 0.f;
        const int oa = o0 + lane, ob = o0 + 32 + lane;
        for (int k = warp; k < SK_SLOTS; k += SK_WARPS) {
            if (!((used >> k) & 1u)) continue;
            const float *wk = (k < 25) ? weight + (int64_t)k * Cin * Cout : rootT;
            const float *ak = A + (size_t)k * Cin * CPB;
            // weights are fetched in batches of 8 rows (16 independent loads in flight) before the FMAs: the
            // loop is otherwise one exposed L2 round trip per row
            for (int c0 = 0; c0 < Cin; c0 += 8) {
                float wa[8], wb[8];
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    const int c = c0 + u;
                    wa[u] = (c < Cin && oa < Cout) ? __ldg(wk + (int64_t)c * Cout + oa) : 0.f;
                    wb[u] = (c < Cin && ob < Cout) ? __ldg(wk + (int64_t)c * Cout + ob) : 0.f;
                }
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    const int c = min(c0 + u, Cin - 1);                  // clamped rows carry zero weights
                    if (CPB % 4 == 0) {
#pragma unroll
                        for (int j4 = 0; j4 < CPB / 4; j4++) {
                            const float4 a4 = *reinterpret_cast<const float4 *>(ak + (size_t)c * CPB + 4 * j4);
                            acc[0][4 * j4 + 0] = fmaf(a4.x, wa[u], acc[0][4 * j4 + 0]); acc[1][4 * j4 + 0] = fmaf(a4.x, wb[u], acc[1][4 * j4 + 0]);
                            acc[0][4 * j4 + 1] = fmaf(a4.y, wa[u], acc[0][4 * j4 + 1]); acc[1][4 * j4 + 1] = fmaf(a4.y, wb[u], acc[1][4 * j4 + 1]);
                            acc[0][4 * j4 + 2] = fmaf(a4.z, wa[u], acc[0][4 * j4 + 2]); acc[1][4 * j4 + 2] = fmaf(a4.z, wb[u], acc[1][4 * j4 + 2]);
                            acc[0][4 * j4 + 3] = fmaf(a4.w, wa[u], acc[0][4 * j4 + 3]); acc[1][4 * j4 + 3] = fmaf(a4.w, wb[u], acc[1][4 * j4 + 3]);
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < CPB; j++) {
                            const float a = ak[(size_t)c * CPB + j];
                            acc[0][j] = fmaf(a, wa[u], acc[0][j]); acc[1][j] = fmaf(a, wb[u], acc[1][j]);
                        }
                    }
                }
            }
        }
        // ---- phase 3: reduce the 8 partial sums, epilogue ---------------------------------------------------------
        __syncthreads();
#pragma unroll
        for (int j = 0; j < CPB; j++) {
            if (oa < Cout) part[((size_t)warp * CPB + j) * Cout + oa] = acc[0][j];
            if (ob < Cout) part[((size_t)warp * CPB + j) * Cout + ob] = acc[1][j];
        }
        __syncthreads();
        const int ow = min(64, Cout - o0);
        for (int i = tid; i < CPB * ow; i += blockDim.x) {
            const int j = i / ow, o = o0 + i % ow;
            const int cell = cell0 + j;
            if (cell >= cells) continue;
            float v = 0.f;
            if (cnt[cell] > 0) {
#pragma unroll
                for (int w2 = 0; w2 < SK_WARPS; w2++) v += part[((size_t)w2 * CPB + j) * Cout + o];
                if (bias) v += bias[o];
                if (scale) v = fmaf(v, scale[o], shift[o]);
                if (skip) v += skip[(int64_t)cell * Cout + o];
                if (relu) v = fmaxf(v, 0.f);
            }
            out[(int64_t)cell * Cout + o] = v;
        }
    }
}

template <int CPB>
static int launch_grid_conv_sk(const dagr_grid_t *gr, const int32_t *cnt, const int32_t *pxy, const uint32_t *mask,
                               const float *xin, int ldin, int Cin, int Cout, const float *weight, const float *rootT, const float *bias,
                               const float *scale, const float *shift, const float *skip, int relu, float den_x, float den_y,
                               float *out, cudaStream_t st)
{
    const int cells = gr->B * gr->ny * gr->nx;
    const size_t a_bytes = (size_t)SK_SLOTS * Cin * CPB * sizeof(float), p_bytes = (size_t)SK_WARPS * CPB * Cout * sizeof(float);
    const size_t smem = (Cout <= 64) ? (a_bytes > p_bytes ? a_bytes : p_bytes) : a_bytes + p_bytes;
    if (smem > 200 * 1024) return -1;
    cudaError_t e = dagr_allow_smem(k_grid_conv_sk<CPB>, smem);
    if (e != cudaSuccess) return -2;
    k_grid_conv_sk<CPB><<<dagr_div_up(cells, CPB), SK_WARPS * 32, smem, st>>>(*gr, cnt, pxy, mask, xin, ldin, Cin, Cout, weight, rootT, bias,
                                                                            scale, shift, skip, relu, den_x, den_y, out);
    return 0;
}

extern "C" int dagr_grid_conv(const dagr_grid_t *gr, const int32_t *cnt, const int32_t *pxy, const uint32_t *mask,
                              const float *xin, int ldin, int Cin, int Cout, const float *weight, const float *rootT,
                              const float *bias, const float *scale, const float *shift, const float *skip, int relu,
                              float den_x, float den_y, float *out, void *stream)
{
    DAGR_CHECK_ARG(gr && Cin > 0 && Cout > 0 && (ldin == 0 || ldin >= Cin), "bad channels");
    if (ldin == 0) ldin = Cin;
    const int cells = gr->B * gr->ny * gr->nx;
    cudaStream_t st = (cudaStream_t)stream;
    // voxels per CTA: enough CTAs to fill every SM, as much weight reuse as shared memory allows
    static int n_sm = 0;
    if (n_sm == 0) {
        int dev = 0;
        DAGR_CUDA(cudaGetDevice(&dev));
        DAGR_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    int rc = -1;
    const size_t per_cell = ((size_t)SK_SLOTS * Cin + (Cout <= 64 ? 0 : (size_t)SK_WARPS * Cout)) * sizeof(float);
    if (cells >= n_sm * 16 * 2 && per_cell * 16 <= 110 * 1024)
        rc = launch_grid_conv_sk<16>(gr, cnt, pxy, mask, xin, ldin, Cin, Cout, weight, rootT, bias, scale, shift, skip, relu, den_x, den_y, out, st);
    if (rc != 0 && cells >= n_sm * 4 && per_cell * 4 <= 160 * 1024)
        rc = launch_grid_conv_sk<4>(gr, cnt, pxy, mask, xin, ldin, Cin, Cout, weight, rootT, bias, scale, shift, skip, relu, den_x, den_y, out, st);
    if (rc != 0)
        rc = launch_grid_conv_sk<1>(gr, cnt, pxy, mask, xin, ldin, Cin, Cout, weight, rootT, bias, scale, shift, skip, relu, den_x, den_y, out, st);
    if (rc != 0) {
        // very wide layers: v1 kernel (one warp per voxel)
        const size_t smem = (size_t)GC_WARPS * GC_SLOTS * Cin * sizeof(float);
        DAGR_CHECK_ARG(smem <= 200 * 1024, "Cin too large for the grid conv kernels");
        DAGR_CUDA(dagr_allow_smem(k_grid_conv, smem));
        k_grid_conv<<<dagr_div_up(cells, GC_WARPS), GC_WARPS * 32, smem, st>>>(
            *gr, cnt, pxy, mask, xin, ldin, Cin, Cout, weight, rootT, bias, scale, shift, skip, relu, den_x, den_y, out);
    }
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// Linear (no bias) + eval BN on valid voxels: the skip branch of ConvBlockWithSkip
// ------------------------------------------------------------------------------------------------
// One CTA per LB_CELLS voxels: their input rows sit in shared memory, thread (o, half) owns output channel o of four
// voxels, so every weight is loaded once per four FMAs and the loads of eight rows are in flight before the FMAs (the
// one-warp-per-voxel form this replaces was a chain of Cin dependent L2 round trips).
#define LB_CELLS 8
__global__ void __launch_bounds__(256)
k_grid_linear_bn(int64_t cells, const int32_t *__restrict__ cnt, const float *__restrict__ xin, int Cin,
                 int Cout, const float *__restrict__ wT, const float *__restrict__ scale,
                 const float *__restrict__ shift, float *__restrict__ out)
{
    extern __shared__ float s_x[];                                       // [LB_CELLS][Cin]
    __shared__ int s_valid[LB_CELLS];
    const int64_t cell0 = (int64_t)blockIdx.x * LB_CELLS;
    for (int i = threadIdx.x; i < LB_CELLS * Cin; i += blockDim.x) {
        const int64_t cell = cell0 + i / Cin;
        s_x[i] = (cell < cells) ? xin[cell * Cin + i % Cin] : 0.f;
    }
    if (threadIdx.x < LB_CELLS) s_valid[threadIdx.x] = (cell0 + threadIdx.x < cells) && cnt[cell0 + threadIdx.x] > 0;
    __syncthreads();
    const int groups = LB_CELLS / 4;
    for (int t = threadIdx.x; t < Cout * groups; t += blockDim.x) {
        const int o = t % Cout, jg = t / Cout;
        const float *x0 = s_x + (size_t)(4 * jg) * Cin;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int c0 = 0; c0 < Cin; c0 += 8) {
            float w[8];
#pragma unroll
            for (int u = 0; u < 8; u++) w[u] = (c0 + u < Cin) ? __ldg(wT + (int64_t)(c0 + u) * Cout + o) : 0.f;
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int c = min(c0 + u, Cin - 1);                      // clamped rows carry zero weights
#pragma unroll
                for (int k = 0; k < 4; k++) acc[k] = fmaf(x0[(size_t)k * Cin + c], w[u], acc[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int64_t cell = cell0 + 4 * jg + k;
            if (cell >= cells) continue;
            float v = 0.f;
            if (s_valid[4 * jg + k]) v = scale ? fmaf(acc[k], scale[o], shift[o]) : acc[k];
            out[cell * Cout + o] = v;
        }
    }
}

extern "C" int dagr_grid_linear_bn(int64_t cells, const int32_t *cnt, const float *xin, int Cin, int Cout,
                                   const float *wT, const float *scale, const float *shift, float *out, void *stream)
{
    DAGR_CHECK_ARG(Cin > 0 && Cout > 0 && (size_t)LB_CELLS * Cin * 4 <= 48 * 1024, "bad channels");
    if (cells <= 0) return DAGR_OK;
    k_grid_linear_bn<<<dagr_div_up(cells, LB_CELLS), 256, (size_t)LB_CELLS * Cin * sizeof(float), (cudaStream_t)stream>>>(
        cells, cnt, xin, Cin, Cout, wT, scale, shift, out);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// pooling between voxel grids (pool2..4)
// ------------------------------------------------------------------------------------------------
__global__ void k_grid_pool(const dagr_grid_t ch, const dagr_grid_t pa, const int32_t *__restrict__ cellx,
                            const int32_t *__restrict__ celly, const int32_t *__restrict__ cnt,
                            const int32_t *__restrict__ pxy, const float *__restrict__ tmean,
                            const float *__restrict__ tmax, const uint32_t *__restrict__ mask,
                            const float *__restrict__ x, int C, int aggr, uint32_t *__restrict__ accmax,
                            double *__restrict__ accsum, double *__restrict__ possum, uint32_t *__restrict__ ptmax,
                            int32_t *__restrict__ pcnt, uint32_t *__restrict__ pmask, int32_t *__restrict__ err)
{
    const int cells = ch.B * ch.ny * ch.nx;
    const int cell = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (cell >= cells || cnt[cell] <= 0) return;
    const int per = ch.ny * ch.nx;
    const int b = cell / per, rem = cell % per, cy = rem / ch.nx, cx = rem % ch.nx;
    const int pper = pa.ny * pa.nx;
    const int px = pxy[2 * cell], py = pxy[2 * cell + 1];
    const int Px = cellx[px], Py = celly[py];
    const int P = b * pper + Py * pa.nx + Px;
    if (lane == 0) {
        atomicAdd(pcnt + P, 1);
        atomicAdd(possum + 3 * (int64_t)P + 0, (double)ch.posxr[px]);
        atomicAdd(possum + 3 * (int64_t)P + 1, (double)ch.posyr[py]);
        atomicAdd(possum + 3 * (int64_t)P + 2, (double)tmean[cell]);
        // t_max of the parent = max over its children of THEIR position t, i.e. the child's mean t (pooling.py:70 reads
        // data.pos[:, -1], which after the previous pooling is pool_pos' mean) -- not the max of the children's t_max
        atomicMax(ptmax + P, enc_ordered(tmean[cell]));
        (void)tmax;
        const uint32_t m = mask[cell];
        uint32_t bits = 0;
        for (int bit = 0; bit < 9; bit++) {
            if (!((m >> bit) & 1u) || bit == 4) continue;
            const int sx = cx + bit % 3 - 1, sy = cy + bit / 3 - 1;
            if (sx < 0 || sy < 0 || sx >= ch.nx || sy >= ch.ny) continue;
            const int src = b * per + sy * ch.nx + sx;
            if (cnt[src] <= 0) continue;
            const int SPx = cellx[pxy[2 * src]], SPy = celly[pxy[2 * src + 1]];
            const int ddx = SPx - Px, ddy = SPy - Py;
            if (ddx == 0 && ddy == 0) continue;                        // self loop dropped (pooling.py:62)
            if (ddx < -1 || ddx > 1 || ddy < -1 || ddy > 1) { atomicExch(err, 1); continue; }
            bits |= 1u << ((ddy + 1) * 3 + (ddx + 1));
        }
        if (bits) atomicOr(pmask + P, bits);
    }
    for (int c = lane; c < C; c += 32) {
        const float v = x[(int64_t)cell * C + c];
        if (aggr == 0) atomicMax(accmax + (int64_t)P * C + c, enc_ordered(v));
        else atomicAdd(accsum + (int64_t)P * C + c, (double)v);
    }
}

extern "C" int dagr_grid_pool(const dagr_grid_t *child, const dagr_grid_t *parent, const int32_t *cellx,
                              const int32_t *celly, const int32_t *cnt, const int32_t *pxy, const float *tmean,
                              const float *tmax, const uint32_t *mask, const float *x, int C, int aggr,
                              uint32_t *accmax, double *accsum, double *possum, uint32_t *ptmax, int32_t *pcnt,
                              uint32_t *pmask, int32_t *err_flag, void *stream)
{
    const int cells = child->B * child->ny * child->nx;
    k_grid_pool<<<dagr_div_up(cells, 4), 128, 0, (cudaStream_t)stream>>>(*child, *parent, cellx, celly, cnt, pxy, tmean, tmax,
                                                                       mask, x, C, aggr, accmax, accsum, possum, ptmax,
                                                                       pcnt, pmask, err_flag);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

__global__ void k_grid_pool_finalize(const dagr_grid_t pa, int C, int aggr, const uint32_t *__restrict__ accmax,
                                     const double *__restrict__ accsum, const double *__restrict__ possum,
                                     const uint32_t *__restrict__ ptmax, const int32_t *__restrict__ pcnt,
                                     int32_t *__restrict__ pxy, float *__restrict__ tmean, float *__restrict__ tmax,
                                     float *__restrict__ x)
{
    const int cells = pa.B * pa.ny * pa.nx;
    const int cell = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (cell >= cells) return;
    const int n = pcnt[cell];
    if (lane == 0) {
        if (n > 0) {
            const float mx = (float)(possum[3 * (int64_t)cell] / (double)n);
            const float my = (float)(possum[3 * (int64_t)cell + 1] / (double)n);
            pxy[2 * cell] = round_to_pixel(mx, pa.W);
            pxy[2 * cell + 1] = round_to_pixel(my, pa.H);
            tmean[cell] = (float)(possum[3 * (int64_t)cell + 2] / (double)n);
            tmax[cell] = dec_ordered(ptmax[cell]);
        } else {
            pxy[2 * cell] = 0; pxy[2 * cell + 1] = 0; tmean[cell] = 0.f; tmax[cell] = 0.f;
        }
    }
    for (int c = lane; c < C; c += 32) {
        float v = 0.f;
        if (n > 0) v = aggr == 0 ? dec_ordered(accmax[(int64_t)cell * C + c])
                                 : (float)(accsum[(int64_t)cell * C + c] / (double)n);
        x[(int64_t)cell * C + c] = v;
    }
}

extern "C" int dagr_grid_pool_finalize(const dagr_grid_t *parent, int C, int aggr, const uint32_t *accmax,
                                       const double *accsum, const double *possum, const uint32_t *ptmax,
                                       const int32_t *pcnt, int32_t *pxy, float *tmean, float *tmax, float *x,
                                       void *stream)
{
    const int cells = parent->B * parent->ny * parent->nx;
    k_grid_pool_finalize<<<dagr_div_up(cells, 4), 128, 0, (cudaStream_t)stream>>>(*parent, C, aggr, accmax, accsum, possum,
                                                                                ptmax, pcnt, pxy, tmean, tmax, x);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// keep_temporal_ordering (pooling.py:69-72)
__global__ void k_temporal_filter(const dagr_grid_t gr, const int32_t *__restrict__ cnt, const float *__restrict__ tmax,
                                  uint32_t *__restrict__ mask)
{
    const int cells = gr.B * gr.ny * gr.nx;
    const int cell = blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= cells || cnt[cell] <= 0) return;
    const int per = gr.ny * gr.nx;
    const int b = cell / per, rem = cell % per, cy = rem / gr.nx, cx = rem % gr.nx;
    uint32_t m = mask[cell], keep = 0;
    for (int bit = 0; bit < 9; bit++) {
        if (!((m >> bit) & 1u) || bit == 4) continue;
        const int sx = cx + bit % 3 - 1, sy = cy + bit / 3 - 1;
        if (sx < 0 || sy < 0 || sx >= gr.nx || sy >= gr.ny) continue;
        const int src = b * per + sy * gr.nx + sx;
        if (cnt[src] > 0 && tmax[cell] > tmax[src]) keep |= 1u << bit;
    }
    mask[cell] = keep;
}

extern "C" int dagr_grid_temporal_filter(const dagr_grid_t *gr, const int32_t *cnt, const float *tmax, uint32_t *mask,
                                         void *stream)
{
    const int cells = gr->B * gr->ny * gr->nx;
    k_temporal_filter<<<dagr_div_up(cells, 128), 128, 0, (cudaStream_t)stream>>>(*gr, cnt, tmax, mask);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// to_dense, decode, NMS
// ------------------------------------------------------------------------------------------------
__global__ void k_to_dense(const dagr_grid_t gr, const int32_t *__restrict__ cnt, const float *__restrict__ x, int C, int ldx,
                           const float *__restrict__ add, float *__restrict__ dense, int64_t total)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int per = gr.ny * gr.nx;
    const int xy = (int)(i % per);
    const int c = (int)((i / per) % C);
    const int b = (int)(i / ((int64_t)per * C));
    const int64_t cell = (int64_t)b * per + xy;
    float v = cnt[cell] > 0 ? x[cell * ldx + c] : 0.f;
    if (add) v += add[i];
    dense[i] = v;
}

extern "C" int dagr_grid_to_dense(const dagr_grid_t *gr, const int32_t *cnt, const float *x, int C, int ldx, const float *add,
                                  float *dense, void *stream)
{
    const int64_t total = (int64_t)gr->B * C * gr->ny * gr->nx;
    if (ldx == 0) ldx = C;
    k_to_dense<<<dagr_div_up(total, 256), 256, 0, (cudaStream_t)stream>>>(*gr, cnt, x, C, ldx, add, dense, total);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

__global__ void k_head_decode(const float *__restrict__ reg, const float *__restrict__ obj, const float *__restrict__ cls,
                              int B, int nc, int h, int w, float stride, int a0, int A, float *__restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int hw = h * w;
    if (i >= B * hw) return;
    const int b = i / hw, a = i % hw, gy = a / w, gx = a % w;
    float *o = out + ((int64_t)b * A + a0 + a) * (5 + nc);
    const float *r = reg + (int64_t)b * 4 * hw + a;
    o[0] = (r[0] + (float)gx) * stride;
    o[1] = (r[hw] + (float)gy) * stride;
    o[2] = expf(r[2 * hw]) * stride;
    o[3] = expf(r[3 * hw]) * stride;
    o[4] = 1.f / (1.f + expf(-obj[(int64_t)b * hw + a]));
    for (int c = 0; c < nc; c++) o[5 + c] = 1.f / (1.f + expf(-cls[((int64_t)b * nc + c) * hw + a]));
}

extern "C" int dagr_head_decode(const float *reg, const float *obj, const float *cls, int B, int nc, int h, int w,
                                int stride, int a0, int A, float *out, void *stream)
{
    k_head_decode<<<dagr_div_up((int64_t)B * h * w, 128), 128, 0, (cudaStream_t)stream>>>(reg, obj, cls, B, nc, h, w,
                                                                                       (float)stride, a0, A, out);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// to_dense (spline_conv.py:80-107) of the three prediction convs + CNN maps (dagr.py:219-222) + collect_outputs /
// decode_outputs (dagr.py:292-312) of one scale in ONE pass: per voxel of the dense head grid
//   reg/obj/cls = (valid ? conv output : 0) + CNN map;  xy = (reg_xy + grid) * stride, wh = exp(reg_wh) * stride,
//   sigmoid(obj), sigmoid(cls)  -> out[b, a0 + cell, 5 + nc]
// (the separate to_dense + head_decode launches, 8 per forward, remain for callers that want the dense maps)
// PLANES: the CNN maps add_* are plane arrays [pl.n][C][ny][nx] and sample b reads plane img_plane(pl, b).
template <bool PLANES>
__global__ void k_head_finish(const dagr_grid_t gr, const int32_t *__restrict__ cnt, const float *__restrict__ cls, int ldc,
                              const float *__restrict__ regobj, int ldr, const float *__restrict__ add_cls,
                              const float *__restrict__ add_reg, const float *__restrict__ add_obj, int nc, float stride, int a0,
                              int A, float *__restrict__ out, const ImgPlanes pl)
{
    const int per = gr.ny * gr.nx;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= gr.B * per) return;
    const int b = i / per, a = i % per, gy = a / gr.nx, gx = a % gr.nx;
    const int bm = PLANES ? img_plane(pl, b) : b;                          // batch index of the CNN maps
    const bool valid = cnt[i] > 0;
    float r[5];
#pragma unroll
    for (int c = 0; c < 5; c++) r[c] = valid ? regobj[(int64_t)i * ldr + c] : 0.f;
    if (add_reg) {
#pragma unroll
        for (int c = 0; c < 4; c++) r[c] += add_reg[((int64_t)bm * 4 + c) * per + a];
    }
    if (add_obj) r[4] += add_obj[(int64_t)bm * per + a];
    float *o = out + ((int64_t)b * A + a0 + a) * (5 + nc);
    o[0] = (r[0] + (float)gx) * stride;
    o[1] = (r[1] + (float)gy) * stride;
    o[2] = expf(r[2]) * stride;
    o[3] = expf(r[3]) * stride;
    o[4] = 1.f / (1.f + expf(-r[4]));
    for (int c = 0; c < nc; c++) {
        float v = valid ? cls[(int64_t)i * ldc + c] : 0.f;
        if (add_cls) v += add_cls[((int64_t)bm * nc + c) * per + a];
        o[5 + c] = 1.f / (1.f + expf(-v));
    }
}

extern "C" int dagr_head_finish(const dagr_grid_t *gr, const int32_t *cnt, const float *cls, int ldc, const float *regobj, int ldr,
                                const float *add_cls, const float *add_reg, const float *add_obj, int nc, int stride, int a0, int A,
                                float *out, void *stream)
{
    DAGR_CHECK_ARG(gr && cls && regobj && ldc >= nc && ldr >= 5, "bad argument");
    const int n = gr->B * gr->ny * gr->nx;
    k_head_finish<false><<<dagr_div_up(n, 128), 128, 0, (cudaStream_t)stream>>>(*gr, cnt, cls, ldc, regobj, ldr, add_cls, add_reg, add_obj,
                                                                              nc, (float)stride, a0, A, out, ImgPlanes{});
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

extern "C" int dagr_head_finish_planes(const dagr_grid_t *gr, const int32_t *cnt, const float *cls, int ldc, const float *regobj,
                                       int ldr, const float *add_cls, const float *add_reg, const float *add_obj, int nc, int stride,
                                       int a0, int A, int nplanes, const int32_t *plane, int plane_stride, float *out, void *stream)
{
    DAGR_CHECK_ARG(gr && cnt && cls && regobj && add_cls && add_reg && add_obj && plane && out, "null argument");
    DAGR_CHECK_ARG(nplanes >= 1, "nplanes must be >= 1");
    DAGR_CHECK_ARG(plane_stride >= 1, "plane_stride must be >= 1");
    DAGR_CHECK_ARG(ldc >= nc && ldr >= 5, "row strides ldc >= nc and ldr >= 5");
    const int n = gr->B * gr->ny * gr->nx;
    k_head_finish<true><<<dagr_div_up(n, 128), 128, 0, (cudaStream_t)stream>>>(*gr, cnt, cls, ldc, regobj, ldr, add_cls, add_reg, add_obj,
                                                                             nc, (float)stride, a0, A, out,
                                                                             ImgPlanes{plane, plane_stride, nplanes});
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

#define NMS_MAX 256
#define NMS_THREADS 1024
// One CTA of 32 warps per image.  The suppression matrix (which lower-ranked candidates would candidate i suppress) is
// built warp-per-candidate: the 32 lanes test 32 lower-ranked candidates at once and a ballot packs the word, so the
// longest dependent chain is ~6 x 6 IoUs instead of 175; ranking and the raw records are one pass over the anchors; only
// the greedy walk over the ranking (torchvision.ops.nms semantics) is serial, over bit words in shared memory.
__global__ void __launch_bounds__(NMS_THREADS)
k_postprocess_nms(const float *__restrict__ pred, int A, int nc, float conf_thre, float nms_thre, float max_dim1,
                  int filtering, float *__restrict__ det, int32_t *__restrict__ ndet)
{
    __shared__ float bx[NMS_MAX][4];     // class-offset boxes used for IoU
    __shared__ float raw[NMS_MAX][6];    // x1, y1, x2, y2, score, class of every anchor
    __shared__ float sc[NMS_MAX];
    __shared__ short order[NMS_MAX];     // candidate ids in descending score order
    __shared__ unsigned char alive[NMS_MAX];
    __shared__ uint32_t supp[NMS_MAX][NMS_MAX / 32];
    __shared__ short s_keep[NMS_MAX];
    __shared__ int ncand, nout;
    const int b = blockIdx.x;
    const float *P = pred + (int64_t)b * A * (5 + nc);
    float *D = det + (int64_t)b * A * 6;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    if (threadIdx.x == 0) ncand = 0;
    __syncthreads();
    // per anchor: xyxy, class max, score, confidence mask (model/utils.py:62-87).  Every rounding step that decides the
    // output is an explicit _rn intrinsic, so nvcc / ptxas cannot contract it into an FMA (w * 0.5 == w / 2 exactly).
    for (int a = threadIdx.x; a < A; a += blockDim.x) {
        const float *p = P + (int64_t)a * (5 + nc);
        const float x1 = __fsub_rn(p[0], __fmul_rn(p[2], 0.5f)), y1 = __fsub_rn(p[1], __fmul_rn(p[3], 0.5f));
        const float x2 = __fadd_rn(p[2], x1), y2 = __fadd_rn(p[3], y1);
        float cc = p[5]; int cl = 0;
        for (int c = 1; c < nc; c++) if (p[5 + c] > cc) { cc = p[5 + c]; cl = c; }
        const float score = __fmul_rn(p[4], cc);
        const bool keep = !filtering || (__fmul_rn(score, cc) >= conf_thre);
        raw[a][0] = x1; raw[a][1] = y1; raw[a][2] = x2; raw[a][3] = y2; raw[a][4] = score; raw[a][5] = (float)cl;
        const float offs = (float)cl * max_dim1;                          // exact integer product: an FMA here is harmless
        bx[a][0] = x1 + offs; bx[a][1] = y1 + offs; bx[a][2] = x2 + offs; bx[a][3] = y2 + offs;
        sc[a] = score;
        alive[a] = keep ? 1 : 0;
    }
    __syncthreads();
    if (!filtering) {
        for (int i = threadIdx.x; i < A * 6; i += blockDim.x) D[i] = raw[i / 6][i % 6];
        if (threadIdx.x == 0) ndet[b] = A;
        return;
    }
    // rank among kept candidates: descending score, ties by anchor index (one warp per anchor, lanes over the others)
    for (int a = warp; a < A; a += nwarps) {
        if (!alive[a]) continue;                                         // warp-uniform
        const float s = sc[a];
        int r = 0;
        for (int j = lane; j < A; j += 32) r += (alive[j] && (sc[j] > s || (sc[j] == s && j < a))) ? 1 : 0;
        r = __reduce_add_sync(0xffffffffu, r);
        if (lane == 0) { order[r] = (short)a; atomicAdd(&ncand, 1); }
    }
    __syncthreads();
    const int n = ncand;
    const int nwords = (n + 31) / 32;
    // suppression words: warp per candidate i, lane k of word wd tests candidate wd*32 + k (only those ranked below i)
    for (int i = warp; i < n; i += nwarps) {
        const int ai = order[i];
        const float ax1 = bx[ai][0], ay1 = bx[ai][1], ax2 = bx[ai][2], ay2 = bx[ai][3];
        const float sa = __fmul_rn(__fsub_rn(ax2, ax1), __fsub_rn(ay2, ay1));
        for (int wd = i >> 5; wd < nwords; wd++) {
            const int k = wd * 32 + lane;
            bool hit = false;
            if (k > i && k < n) {
                // torchvision's CPU IoU, every step rounded on its own: with plain operators nvcc turned sa + sb into
                // fma(dx_b, dy_b, sa), which flips the decision for pairs within an ulp of nms_thre
                const int aj = order[k];
                const float l = fmaxf(ax1, bx[aj][0]), t = fmaxf(ay1, bx[aj][1]);
                const float r = fminf(ax2, bx[aj][2]), bt = fminf(ay2, bx[aj][3]);
                const float iw = fmaxf(__fsub_rn(r, l), 0.f), ih = fmaxf(__fsub_rn(bt, t), 0.f);
                const float inter = __fmul_rn(iw, ih);
                const float sb = __fmul_rn(__fsub_rn(bx[aj][2], bx[aj][0]), __fsub_rn(bx[aj][3], bx[aj][1]));
                hit = __fdiv_rn(inter, __fsub_rn(__fadd_rn(sa, sb), inter)) > nms_thre;
            }
            const uint32_t bits = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) supp[i][wd] = bits;
        }
    }
    __syncthreads();
    // greedy walk in score order: warp 0, lane wd keeps word wd of the dead mask
    if (warp == 0) {
        uint32_t dead = 0;
        int m = 0;
        for (int i = 0; i < n; i++) {
            const uint32_t dw = __shfl_sync(0xffffffffu, dead, i >> 5);
            if ((dw >> (i & 31)) & 1u) continue;                         // warp-uniform
            if (lane == 0) s_keep[m] = order[i];
            m++;
            if (lane < nwords && lane >= (i >> 5)) dead |= supp[i][lane];
        }
        if (lane == 0) nout = m;
    }
    __syncthreads();
    // survivors in score order, zero padding behind them
    for (int i = threadIdx.x; i < A * 6; i += blockDim.x) D[i] = (i / 6 < nout) ? raw[s_keep[i / 6]][i % 6] : 0.f;
    if (threadIdx.x == 0) ndet[b] = nout;
}

extern "C" int dagr_postprocess_nms(const float *pred, int B, int A, int nc, float conf_thre, float nms_thre, int width,
                                    int height, int filtering, float *det, int32_t *ndet, void *stream)
{
    DAGR_CHECK_ARG(pred && det && ndet, "null pred / det / ndet");
    DAGR_CHECK_ARG(nc >= 1, "nc must be >= 1 (a row is cx, cy, w, h, obj and at least one class score)");
    DAGR_CHECK_ARG(A > 0 && A <= NMS_MAX, "A must be in [1,256] (two-scale DAGR heads have 175 anchors)");
    DAGR_CHECK_ARG(B >= 0, "B must be >= 0");
    if (B == 0) return DAGR_OK;
    const float max_dim1 = (float)((width > height ? width : height) + 1);
    k_postprocess_nms<<<B, NMS_THREADS, 0, (cudaStream_t)stream>>>(pred, A, nc, conf_thre, nms_thre, max_dim1, filtering, det, ndet);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// a8 sample_features: 3-D bilinear grid_sample, align_corners=True, zero padding (net.py:193-221)
// PLANES: img_in is a plane array [pl.n][C][h][w]; node i samples plane img_plane(pl, bidx[i]) as a batch of one.
// MT: the map format (common.cuh: float = NCHW, __nv_bfloat16 = NHWC, where the lanes' channels of a tap are one coalesced run).
// ------------------------------------------------------------------------------------------------
template <bool PLANES, typename MT = float>
__global__ void k_sample_features(const MT *__restrict__ img_in, int Bi_in, int C, int h, int w,
                                  const float *__restrict__ posx, const float *__restrict__ posy,
                                  const int32_t *__restrict__ bidx, int64_t n, float width, float height,
                                  float *__restrict__ out, int ldo, int c0, const ImgPlanes pl)
{
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const int Bi = PLANES ? 1 : Bi_in;
    const MT *__restrict__ img = PLANES ? img_in + (int64_t)img_plane(pl, bidx[i]) * C * h * w : img_in;
    // normalise exactly as _sample_features does, then unnormalise as grid_sample(align_corners=True)
    float gx = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fmul_rn(posx[i], width)), width - 1.f), 1.f);
    float gy = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fmul_rn(posy[i], height)), height - 1.f), 1.f);
    const float bs = (float)(Bi > 1 ? Bi : 2);
    float gz = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, PLANES ? 0.f : (float)bidx[i]), bs - 1.f), 1.f);
    const float ix = __fmul_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f), (float)(w - 1));
    const float iy = __fmul_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f), (float)(h - 1));
    const float iz = __fmul_rn(__fmul_rn(__fadd_rn(gz, 1.f), 0.5f), (float)(Bi - 1));
    const float x0f = floorf(ix), y0f = floorf(iy), z0f = floorf(iz);
    const int x0 = (int)x0f, y0 = (int)y0f, z0 = (int)z0f;
    const float tx = ix - x0f, ty = iy - y0f, tz = iz - z0f;
    for (int c = lane; c < C; c += 32) {
        float acc = 0.f;
#pragma unroll
        for (int dz = 0; dz < 2; dz++) {
            const int z = z0 + dz;
            const float wz = dz ? tz : 1.f - tz;
            if (z < 0 || z >= Bi) continue;
#pragma unroll
            for (int dy = 0; dy < 2; dy++) {
                const int y = y0 + dy;
                const float wy = dy ? ty : 1.f - ty;
                if (y < 0 || y >= h) continue;
#pragma unroll
                for (int dx = 0; dx < 2; dx++) {
                    const int x = x0 + dx;
                    const float wx = dx ? tx : 1.f - tx;
                    if (x < 0 || x >= w) continue;
                    acc += map_ld(img, C, h, w, z, c, y, x) * (wx * wy * wz);
                }
            }
        }
        out[i * ldo + c0 + c] = acc;
    }
}

extern "C" int dagr_sample_features(const float *img, int Bi, int C, int h, int w, const float *posx, const float *posy,
                                    const int32_t *bidx, int64_t n, int width, int height, float *out, int ldo, int c0,
                                    void *stream)
{
    if (n <= 0) return DAGR_OK;
    k_sample_features<false><<<dagr_div_up(n, 4), 128, 0, (cudaStream_t)stream>>>(img, Bi, C, h, w, posx, posy, bidx, n,
                                                                                (float)width, (float)height, out, ldo, c0, ImgPlanes{});
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

extern "C" int dagr_sample_features_planes(const float *img, int nplanes, const int32_t *plane, int plane_stride, int C, int h, int w,
                                           const float *posx, const float *posy, const int32_t *bidx, int64_t n, int width, int height,
                                           float *out, int ldo, int c0, void *stream)
{
    DAGR_CHECK_ARG(img && posx && posy && bidx && out && plane, "null argument");
    DAGR_CHECK_ARG(nplanes >= 1, "nplanes must be >= 1");
    DAGR_CHECK_ARG(plane_stride >= 1, "plane_stride must be >= 1");
    DAGR_CHECK_ARG(n >= 0 && n < (1ll << 31), "N out of range");
    if (n == 0) return DAGR_OK;
    k_sample_features<true><<<dagr_div_up(n, 4), 128, 0, (cudaStream_t)stream>>>(img, 1, C, h, w, posx, posy, bidx, n, (float)width,
                                                                               (float)height, out, ldo, c0,
                                                                               ImgPlanes{plane, plane_stride, nplanes});
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// bf16 NHWC forms (include/dagr_b200.h): the same kernel with MT = __nv_bfloat16
extern "C" int dagr_sample_features_bf16(const void *img, int Bi, int C, int h, int w, const float *posx, const float *posy,
                                         const int32_t *bidx, int64_t n, int width, int height, float *out, int ldo, int c0,
                                         void *stream)
{
    DAGR_CHECK_ARG(img && posx && posy && bidx && out, "null argument");
    DAGR_CHECK_ARG(n >= 0 && n < (1ll << 31), "N out of range");
    DAGR_CHECK_ARG(Bi >= 1 && C >= 1 && h >= 1 && w >= 1, "the map must have Bi, C, h, w >= 1");
    if (n == 0) return DAGR_OK;
    k_sample_features<false, __nv_bfloat16><<<dagr_div_up(n, 4), 128, 0, (cudaStream_t)stream>>>(
        static_cast<const __nv_bfloat16 *>(img), Bi, C, h, w, posx, posy, bidx, n, (float)width, (float)height, out, ldo, c0, ImgPlanes{});
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

extern "C" int dagr_sample_features_planes_bf16(const void *img, int nplanes, const int32_t *plane, int plane_stride, int C, int h, int w,
                                                const float *posx, const float *posy, const int32_t *bidx, int64_t n, int width,
                                                int height, float *out, int ldo, int c0, void *stream)
{
    DAGR_CHECK_ARG(img && posx && posy && bidx && out && plane, "null argument");
    DAGR_CHECK_ARG(nplanes >= 1, "nplanes must be >= 1");
    DAGR_CHECK_ARG(plane_stride >= 1, "plane_stride must be >= 1");
    DAGR_CHECK_ARG(n >= 0 && n < (1ll << 31), "N out of range");
    DAGR_CHECK_ARG(C >= 1 && h >= 1 && w >= 1, "the map must have C, h, w >= 1");
    if (n == 0) return DAGR_OK;
    k_sample_features<true, __nv_bfloat16><<<dagr_div_up(n, 4), 128, 0, (cudaStream_t)stream>>>(
        static_cast<const __nv_bfloat16 *>(img), 1, C, h, w, posx, posy, bidx, n, (float)width, (float)height, out, ldo, c0,
        ImgPlanes{plane, plane_stride, nplanes});
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}
