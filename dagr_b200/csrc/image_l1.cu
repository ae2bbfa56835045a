// image_l1.cu -- event-level image fusion (use_image): bilinear sampling of ResNet feature maps at the
// events (net.py:15-17,193-221), conv_block1.conv_block1 on 1+16+2 input channels, and the per-voxel max
// of the 64-channel samples that are concatenated before pool1 (net.py:128-131).  sm_90a.
#include "common.cuh"
#include <type_traits>

// channel c of the map sampled at q, read through the read-only path
template <typename MT>
__device__ __forceinline__ float bilin_sample(const MT *__restrict__ img, int Bi, int C, int h, int w, int c, const Bilin &q)
{
    float acc = 0.f;
    bilin_taps(q, Bi, h, w, [&](const BilinTap &t) { acc += map_ldg(img, C, h, w, t.z, c, t.y, t.x) * t.w(); });
    return acc;
}

// x0[chunk][p][8] = the 16 image channels sampled at the event (two 8-channel chunks); the two 16-byte halves of a row are
// swapped when XA_SWZ(p), like xa, so that the staged conv kernel (conv_l1.cu) reads both with the same row addressing.
// (polarity, x/W, y/H) -- the other three inputs of conv_block1.conv_block1 -- need no gather and are handled by the probe kernel.
// live = start of the sort (or NULL): only positions p < start[g.NK] (the live total) are sampled.  In ring mode N is the ring
// capacity and the sorted positions at or beyond the live total hold stale or never-written xyb words, whose x / y would index
// past posx0 / posy0; the rows they would fill are never read (conv_a_image, conv_b and voxel_sample_max walk the voxels'
// [start[cell], start[cell+1]) ranges, which lie below the total), so they are simply skipped.  live == NULL: the bound is N.
// PLANES: img0 is a plane array [pl.n][16][h][w] and the event of sample b samples plane img_plane(pl, b) as a batch of one.
// MT: the map format (common.cuh: float = NCHW, __nv_bfloat16 = NHWC).
template <bool PLANES, typename MT>
__global__ void k_l1_x0_image(const dagr_geom_t g, int64_t N, const int32_t *__restrict__ live, const uint32_t *__restrict__ xyb,
                              const MT *__restrict__ img0, int h, int w, float *__restrict__ x0, const ImgPlanes pl)
{
    // 4 threads per node: thread q computes image channels 4q..4q+3 = one 16-byte chunk of a row
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t p = t >> 2;
    const int q = (int)(t & 3);
    if (p >= (live != nullptr ? min((int64_t)__ldg(live + g.NK), N) : N)) return;
    const uint32_t wd = xyb[p];
    const int x = wd & 0xfff, y = (wd >> 12) & 0xfff, b = wd >> 24;
    const float px = g.posx0[x], py = g.posy0[y];
    const int Bi = PLANES ? 1 : g.B;
    const MT *img = PLANES ? img0 + (int64_t)img_plane(pl, b) * 16 * h * w : img0;
    const Bilin bl = bilin_setup(px, py, PLANES ? 0 : b, (float)g.W, (float)g.H, Bi, h, w);
    float f[4];
#pragma unroll
    for (int k = 0; k < 4; k++) f[k] = bilin_sample(img, Bi, 16, h, w, 4 * q + k, bl);
    float4 *dst = reinterpret_cast<float4 *>(x0 + ((int64_t)(q >> 1) * N + p) * 8);
    dst[(q & 1) ^ XA_SWZ(p)] = make_float4(f[0], f[1], f[2], f[3]);
}

// The checks and the launch of every x0 form.  live: the form bounds x0 by the live total start[g.NK] (ring and plane forms),
// so start must not be NULL; the unbounded forms pass start = NULL.  The fp32 forms pass C = 16 (their NCHW tap has 16 channels
// by definition), the bf16 forms the caller's C.  feat_s is not an input of any form.
template <bool PLANES, typename MT>
static int x0_image(const char *who, const dagr_geom_t *g, int64_t N, bool live, const int32_t *start, const uint32_t *xyb,
                    const void *img0, int C, int h, int w, const ImgPlanes pl, float *x0, void *stream)
{
    DAGR_CHECK_ARG_AS(who, g && (start || !live) && xyb && img0 && (pl.plane || !PLANES) && x0, "null argument (only feat_s may be NULL)");
    if (PLANES) {
        DAGR_CHECK_ARG_AS(who, pl.n >= 1, "nplanes must be >= 1");
        DAGR_CHECK_ARG_AS(who, pl.stride >= 1, "plane_stride must be >= 1");
    }
    DAGR_CHECK_ARG_AS(who, N >= 0 && N < (1ll << 31), "N out of range");
    DAGR_CHECK_ARG_AS(who, C == 16 && h >= 1 && w >= 1, "the conv1 tap must have 16 channels and h, w >= 1");
    if (N == 0) return DAGR_OK;
    k_l1_x0_image<PLANES, MT><<<dagr_div_up(4 * N, 256), 256, 0, (cudaStream_t)stream>>>(
        *g, N, start, xyb, static_cast<const MT *>(img0), h, w, x0, pl);
    DAGR_CHECK_LAUNCH_AS(who);
    return DAGR_OK;
}

extern "C" int dagr_l1_x0_image(const dagr_geom_t *g, int64_t N, const uint32_t *xyb, const float * /*feat_s*/, const float *img0,
                                int h, int w, float *x0, void *stream)
{
    return x0_image<false, float>(__func__, g, N, false, nullptr, xyb, img0, 16, h, w, ImgPlanes{}, x0, stream);
}

extern "C" int dagr_l1_x0_image_live(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float * /*feat_s*/,
                                     const float *img0, int h, int w, float *x0, void *stream)
{
    return x0_image<false, float>(__func__, g, N, true, start, xyb, img0, 16, h, w, ImgPlanes{}, x0, stream);
}

extern "C" int dagr_l1_x0_image_planes(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float * /*feat_s*/,
                                       const float *img0, int h, int w, int nplanes, const int32_t *plane, int plane_stride, float *x0,
                                       void *stream)
{
    return x0_image<true, float>(__func__, g, N, true, start, xyb, img0, 16, h, w, ImgPlanes{plane, plane_stride, nplanes}, x0, stream);
}

// bf16 NHWC forms (include/dagr_b200.h): the same kernel with the map loader of MT = __nv_bfloat16
extern "C" int dagr_l1_x0_image_bf16(const dagr_geom_t *g, int64_t N, const uint32_t *xyb, const float * /*feat_s*/, const void *img0,
                                     int C, int h, int w, float *x0, void *stream)
{
    return x0_image<false, __nv_bfloat16>(__func__, g, N, false, nullptr, xyb, img0, C, h, w, ImgPlanes{}, x0, stream);
}

extern "C" int dagr_l1_x0_image_live_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                                          const float * /*feat_s*/, const void *img0, int C, int h, int w, float *x0, void *stream)
{
    return x0_image<false, __nv_bfloat16>(__func__, g, N, true, start, xyb, img0, C, h, w, ImgPlanes{}, x0, stream);
}

extern "C" int dagr_l1_x0_image_planes_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                                            const float * /*feat_s*/, const void *img0, int C, int h, int w, int nplanes, const int32_t *plane,
                                            int plane_stride, float *x0, void *stream)
{
    return x0_image<true, __nv_bfloat16>(__func__, g, N, true, start, xyb, img0, C, h, w, ImgPlanes{plane, plane_stride, nplanes}, x0,
                                         stream);
}

// ------------------------------------------------------------------------------------------------
// per-voxel max of image features sampled at the voxel's events (net.py:128-131 before pool1): one CTA per voxel.
// All events of a voxel sample a small window of the feature map (voxel extent x map/sensor scale, + 1), so the window
// of both batch planes the trilinear sample can touch is staged in shared memory once ([z][y][x][C], channels
// innermost -> conflict-free), and every (event, channel) sample reads shared memory only.  The taps are bilin_taps'
// (common.cuh), i.e. the oracle's.  Windows that do not fit fall back to global taps (bilin_sample).
// ------------------------------------------------------------------------------------------------
#define VS_THREADS 128

// channel c sampled at q from the staged window [z - zb][y - yb][x - xb][C]
__device__ __forceinline__ float vs_sample(const float *s_patch, int Bi, int C, int h, int w, int c, const Bilin &q, int zb, int yb,
                                           int xb, int ph, int pw)
{
    float acc = 0.f;
    bilin_taps(q, Bi, h, w, [&](const BilinTap &t) {
        acc += s_patch[(((t.z - zb) * ph + (t.y - yb)) * pw + (t.x - xb)) * C + c] * t.w();
    });
    return acc;
}

// MEAN: the pooling's aggregation (pooling.py:74-77, args.pooling_aggr); max in every shipped config
template <bool MEAN> __device__ __forceinline__ float vs_comb(float a, float b) { return MEAN ? a + b : fmaxf(a, b); }

// INC (incremental stream step, max only): persist f32[cells][C] holds the running per-voxel max of the samples between steps
// (the reference's async pool1 keeps a running max of the concatenated x, max_pool.py:59-62).  min_idx > 0: only events with
// arrival index ti[p].y >= min_idx are sampled and their max is combined with persist; a voxel without such events copies
// persist and stages nothing.  min_idx == 0 samples every event (the bits of the plain instance) and seeds persist.
// PLANES: img is a plane array [pl.n][C][h][w]; a voxel of sample b samples plane img_plane(pl, b) as a batch of one, so its
// window is staged from that one plane (pz = 1).
// MT: the map format (common.cuh: float = NCHW, __nv_bfloat16 = NHWC).  The window is staged as fp32 in either, so the sampling
// below reads the same shared memory in both.
template <bool MEAN, bool INC, bool PLANES, typename MT>
__global__ void __launch_bounds__(VS_THREADS)
k_voxel_sample_max(const dagr_geom_t g, const int32_t *__restrict__ start, const uint32_t *__restrict__ xyb,
                   const int2 *__restrict__ ti, const MT *__restrict__ img_in, int C, int h, int w, const int min_idx,
                   float *__restrict__ persist, float *__restrict__ xg, int ldx, int c0, const ImgPlanes pl)
{
    __shared__ float s_m[VS_THREADS / 32][128];
    __shared__ __align__(16) float s_patch[DAGR_VS_SMEM_FLOATS];
    const int cell = blockIdx.x;
    const int per = g.ny1 * g.nx1;
    const int b = cell / per, rem = cell % per, cy = rem / g.nx1, cx = rem % g.nx1;
    const int p0 = start[(int64_t)cell * g.CP], p1 = start[(int64_t)(cell + 1) * g.CP];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (p1 == p0) {                                                       // block-uniform
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            xg[(int64_t)cell * ldx + c0 + c] = 0.f;
            if (INC && min_idx <= 0) persist[(int64_t)cell * C + c] = -INFINITY;
        }
        return;
    }
    if (INC && min_idx > 0) {
        bool any = false;
        for (int p = p0 + (int)threadIdx.x; p < p1 && !any; p += blockDim.x) any = __ldg(&ti[p].y) >= min_idx;
        if (!__syncthreads_or(any)) {                                     // nothing new in this voxel: keep its running max
            for (int c = threadIdx.x; c < C; c += blockDim.x) xg[(int64_t)cell * ldx + c0 + c] = persist[(int64_t)cell * C + c];
            return;
        }
    }
    // the events sampled in this launch (INC: the new ones)
    auto take = [&](int p) { return !INC || min_idx <= 0 || __ldg(&ti[p].y) >= min_idx; };
    // the voxel's result for channel c: INC combines it with the running max and stores it back
    auto finish = [&](int c, float v) {
        if (INC) {
            float *pc = persist + (int64_t)cell * C + c;
            if (min_idx > 0) v = fmaxf(v, *pc);
            *pc = v;
        }
        xg[(int64_t)cell * ldx + c0 + c] = v;
    };
    // the sampled batch: sample b of the g.B planes of img, or (PLANES) the one plane of sample b as a batch of one (its depth
    // coordinate and batch size are spelled out at each use below: a local copy of g.B changes the plain instances' allocation)
    const MT *__restrict__ img = PLANES ? img_in + (int64_t)img_plane(pl, b) * C * h * w : img_in;
    // window of the map this voxel's pixels can touch: the sample coordinates are monotone in x / y, so the corner
    // pixels bound it (same arithmetic as the per-event set-up)
    const Bilin lo = bilin_setup(g.posx0[g.vx0[cx]], g.posy0[g.vy0[cy]], PLANES ? 0 : b, (float)g.W, (float)g.H, PLANES ? 1 : g.B, h, w);
    const Bilin hi = bilin_setup(g.posx0[g.vx0[cx + 1] - 1], g.posy0[g.vy0[cy + 1] - 1], PLANES ? 0 : b, (float)g.W, (float)g.H, PLANES ? 1 : g.B, h, w);
    const int xb = max(lo.x0, 0), yb = max(lo.y0, 0), zb = max(lo.z0, 0);
    const int xe = min(hi.x0 + 1, w - 1), ye = min(hi.y0 + 1, h - 1), ze = min(lo.z0 + 1, (PLANES ? 1 : g.B) - 1);
    const int pw = xe - xb + 1, ph = ye - yb + 1, pz = ze - zb + 1;
    const bool staged = pw > 0 && ph > 0 && pz > 0 && (int64_t)pz * ph * pw * C <= DAGR_VS_SMEM_FLOATS;   // block-uniform
    if (staged) {
        const int tot = pz * ph * pw * C;
        if constexpr (std::is_same<MT, float>::value) {
            for (int i = threadIdx.x; i < tot; i += blockDim.x) {
                const int x = i % pw, r1 = i / pw, y = r1 % ph, r2 = r1 / ph, c = r2 % C, z = r2 / C;      // x fastest: coalesced
                s_patch[((z * ph + y) * pw + x) * C + c] = __ldg(img + (((int64_t)(zb + z) * C + c) * h + yb + y) * w + xb + x);
            }
        } else {
            // NHWC: the window has the map's own element order, one contiguous run of pw * C per (z, y) row
            const int run = pw * C;
            for (int i = threadIdx.x; i < tot; i += blockDim.x) {
                const int k = i % run, r = i / run, y = r % ph, z = r / ph;
                s_patch[i] = __bfloat162float(__ldg(img + (((int64_t)(zb + z) * h + yb + y) * w + xb) * C + k));
            }
        }
        __syncthreads();
    }
    // fast path: C/8 lanes per event (8 channels = two 16-byte shared loads per tap and lane), 32/(C/8) events per warp;
    // the 8 trilinear tap weights are computed once per lane and reused for its 8 channels
    const int lpe = C >> 3;                                               // lanes per event
    if (staged && (C & 7) == 0 && C <= 128 && lpe >= 1 && (lpe & (lpe - 1)) == 0) {          // block-uniform
        const int epw = 32 / lpe, sub = lane / lpe, cl = (lane % lpe) * 8;
        float m[8];
#pragma unroll
        for (int k = 0; k < 8; k++) m[k] = MEAN ? 0.f : -INFINITY;
        for (int pb = p0 + wid * epw; pb < p1; pb += (VS_THREADS / 32) * epw) {
            const int p = pb + sub;
            if (p < p1 && take(p)) {
                const uint32_t wd = xyb[p];
                const int x = wd & 0xfff, y = (wd >> 12) & 0xfff;
                const Bilin q = bilin_setup(g.posx0[x], g.posy0[y], PLANES ? 0 : b, (float)g.W, (float)g.H, PLANES ? 1 : g.B, h, w);
                float acc[8];
#pragma unroll
                for (int k = 0; k < 8; k++) acc[k] = 0.f;
                bilin_taps(q, PLANES ? 1 : g.B, h, w, [&](const BilinTap &t) {
                    const float wgt = t.w();
                    const float4 *src = reinterpret_cast<const float4 *>(s_patch + (((t.z - zb) * ph + (t.y - yb)) * pw + (t.x - xb)) * C + cl);
                    const float4 v0 = src[0], v1 = src[1];
                    acc[0] += v0.x * wgt; acc[1] += v0.y * wgt; acc[2] += v0.z * wgt; acc[3] += v0.w * wgt;
                    acc[4] += v1.x * wgt; acc[5] += v1.y * wgt; acc[6] += v1.z * wgt; acc[7] += v1.w * wgt;
                });
#pragma unroll
                for (int k = 0; k < 8; k++) m[k] = vs_comb<MEAN>(m[k], acc[k]);
            }
        }
        // lanes with the same channel block sit lpe apart
        for (int d = lpe; d < 32; d <<= 1)
#pragma unroll
            for (int k = 0; k < 8; k++) m[k] = vs_comb<MEAN>(m[k], __shfl_xor_sync(0xffffffffu, m[k], d));
        float *s_mm = &s_m[0][0];                                          // [warps][128]
        if (lane < lpe) {
#pragma unroll
            for (int k = 0; k < 8; k++) s_mm[wid * 128 + cl + k] = m[k];
        }
        __syncthreads();
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            float v = s_mm[c];
            for (int w2 = 1; w2 < VS_THREADS / 32; w2++) v = vs_comb<MEAN>(v, s_mm[w2 * 128 + c]);
            finish(c, MEAN ? __fdiv_rn(v, (float)(p1 - p0)) : v);
        }
        return;
    }
    for (int cb = 0; cb < C; cb += 128) {
        const float ident = MEAN ? 0.f : -INFINITY;
        float m[4] = {ident, ident, ident, ident};
        for (int p = p0 + wid; p < p1; p += VS_THREADS / 32) {
            if (!take(p)) continue;
            const uint32_t wd = xyb[p];
            const int x = wd & 0xfff, y = (wd >> 12) & 0xfff;
            const Bilin bl = bilin_setup(g.posx0[x], g.posy0[y], PLANES ? 0 : b, (float)g.W, (float)g.H, PLANES ? 1 : g.B, h, w);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int c = cb + lane + 32 * k;
                if (c < C)
                    m[k] = vs_comb<MEAN>(m[k], staged ? vs_sample(s_patch, PLANES ? 1 : g.B, C, h, w, c, bl, zb, yb, xb, ph, pw)
                                                      : bilin_sample(img, PLANES ? 1 : g.B, C, h, w, c, bl));
            }
        }
#pragma unroll
        for (int k = 0; k < 4; k++) s_m[wid][lane + 32 * k] = m[k];
        __syncthreads();
        const int c = cb + threadIdx.x;
        if (c < C) {
            float v = s_m[0][threadIdx.x];
            for (int w2 = 1; w2 < VS_THREADS / 32; w2++) v = vs_comb<MEAN>(v, s_m[w2][threadIdx.x]);
            finish(c, MEAN ? __fdiv_rn(v, (float)(p1 - p0)) : v);
        }
        __syncthreads();
    }
}

// The checks and the launch of every voxel form; pool_mean selects MEAN.  The INC forms pass ti, min_idx and persist, the others
// NULL, 0 and NULL.  Every form launches at N == 0 too: the kernel writes the zeros of the empty voxels.
template <bool INC, bool PLANES, typename MT>
static int voxel_sample(const char *who, const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                        const void *img_in, int C, int h, int w, int min_idx, float *persist, const ImgPlanes pl, float *xg, int ldx,
                        int c0, int pool_mean, void *stream)
{
    DAGR_CHECK_ARG_AS(who, g && start && xyb && (ti || !INC) && img_in && (persist || !INC) && (pl.plane || !PLANES) && xg, "null argument");
    if (INC) DAGR_CHECK_ARG_AS(who, min_idx >= 0, "min_idx must be >= 0");
    if (PLANES) {
        DAGR_CHECK_ARG_AS(who, pl.n >= 1, "nplanes must be >= 1");
        DAGR_CHECK_ARG_AS(who, pl.stride >= 1, "plane_stride must be >= 1");
    }
    DAGR_CHECK_ARG_AS(who, N >= 0 && N < (1ll << 31), "N out of range");
    DAGR_CHECK_ARG_AS(who, h >= 1 && w >= 1, "the map must have h, w >= 1");
    DAGR_CHECK_ARG_AS(who, C >= 1 && c0 >= 0 && c0 + C <= ldx, "the channels [c0, c0 + C) must lie within the row stride ldx");
    if (INC) DAGR_CHECK_ARG_AS(who, !pool_mean, "pool_mean: the running per-voxel aggregate of the event stream is a max (max_pool.py:59-62)");
    const int cells = g->B * g->ny1 * g->nx1;
    const cudaStream_t st = (cudaStream_t)stream;
    const MT *img = static_cast<const MT *>(img_in);
    // MEAN never meets INC (refused above), and naming that pair would compile an instance that no form launches
    if (!INC && pool_mean) k_voxel_sample_max<true, false, PLANES, MT><<<cells, VS_THREADS, 0, st>>>(*g, start, xyb, (const int2 *)ti, img, C,
                                                                                                   h, w, min_idx, persist, xg, ldx, c0, pl);
    else                   k_voxel_sample_max<false, INC, PLANES, MT><<<cells, VS_THREADS, 0, st>>>(*g, start, xyb, (const int2 *)ti, img, C,
                                                                                                  h, w, min_idx, persist, xg, ldx, c0, pl);
    DAGR_CHECK_LAUNCH_AS(who);
    return DAGR_OK;
}

extern "C" int dagr_voxel_sample_max(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *img,
                                     int C, int h, int w, float *xg, int ldx, int c0, int pool_mean, void *stream)
{
    return voxel_sample<false, false, float>(__func__, g, N, start, xyb, nullptr, img, C, h, w, 0, nullptr, ImgPlanes{}, xg, ldx, c0,
                                             pool_mean, stream);
}

extern "C" int dagr_voxel_sample_max_inc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                                         const float *img, int C, int h, int w, int min_idx, float *persist, float *xg, int ldx, int c0,
                                         int pool_mean, void *stream)
{
    return voxel_sample<true, false, float>(__func__, g, N, start, xyb, ti, img, C, h, w, min_idx, persist, ImgPlanes{}, xg, ldx, c0,
                                            pool_mean, stream);
}

extern "C" int dagr_voxel_sample_max_planes(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *img,
                                            int C, int h, int w, int nplanes, const int32_t *plane, int plane_stride, float *xg, int ldx,
                                            int c0, int pool_mean, void *stream)
{
    return voxel_sample<false, true, float>(__func__, g, N, start, xyb, nullptr, img, C, h, w, 0, nullptr,
                                            ImgPlanes{plane, plane_stride, nplanes}, xg, ldx, c0, pool_mean, stream);
}

// bf16 NHWC forms (include/dagr_b200.h): the same kernel with MT = __nv_bfloat16
extern "C" int dagr_voxel_sample_max_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const void *img,
                                          int C, int h, int w, float *xg, int ldx, int c0, int pool_mean, void *stream)
{
    return voxel_sample<false, false, __nv_bfloat16>(__func__, g, N, start, xyb, nullptr, img, C, h, w, 0, nullptr, ImgPlanes{}, xg, ldx,
                                                     c0, pool_mean, stream);
}

extern "C" int dagr_voxel_sample_max_inc_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                                              const void *img, int C, int h, int w, int min_idx, float *persist, float *xg, int ldx, int c0,
                                              int pool_mean, void *stream)
{
    return voxel_sample<true, false, __nv_bfloat16>(__func__, g, N, start, xyb, ti, img, C, h, w, min_idx, persist, ImgPlanes{}, xg, ldx,
                                                    c0, pool_mean, stream);
}

extern "C" int dagr_voxel_sample_max_planes_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const void *img,
                                                 int C, int h, int w, int nplanes, const int32_t *plane, int plane_stride, float *xg,
                                                 int ldx, int c0, int pool_mean, void *stream)
{
    return voxel_sample<false, true, __nv_bfloat16>(__func__, g, N, start, xyb, nullptr, img, C, h, w, 0, nullptr,
                                                    ImgPlanes{plane, plane_stride, nplanes}, xg, ldx, c0, pool_mean, stream);
}
