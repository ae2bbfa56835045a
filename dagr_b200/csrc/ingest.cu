// ingest.cu -- event ingest on the device (SURVEY 8(f) rank 1): the steps between the raw DSEC stream and the graph
// builder, which the reference runs on the CPU (numba / numpy) per sample:
//   * 2x event down-sampler            scripts/downsample_events.py:91-124
//   * window slice, crop, relative t   src/dagr/data/dsec_data.py:141-147,177-179
//   * int16/int32 casts, fp32 normalise, denormalise   data/utils.py:6-20, utils/buffers.py:33-44, ev_tgn.py:11-16
// producing directly the int32 (batch, pos) + polarity arrays that dagr_graph_sort consumes.
#include "common.cuh"

// ------------------------------------------------------------------------------------------------
// down-sampler.  The reference walks the events of a chunk in time order and keeps one signed fp32 accumulator per
// output pixel: += p/(fx*fy); when |acc| >= 1 the event passes and acc -= p.  Events of different output pixels never
// interact, so: bin the events by output pixel (histogram -> scan -> scatter -> in-bin rank by arrival index = a stable
// counting sort), then one thread per pixel replays ITS events in time order with the reference's arithmetic.
// ------------------------------------------------------------------------------------------------
__global__ void k_ds_hist(const uint16_t *__restrict__ x, const uint16_t *__restrict__ y, int64_t N, int fx, int fy, int ow,
                          int oh, int32_t *__restrict__ cell, int32_t *__restrict__ count)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int xl = min((int)x[i] / fx, ow - 1), yl = min((int)y[i] / fy, oh - 1);   // the reference would index out of bounds
    const int c = yl * ow + xl;
    cell[i] = c;
    atomicAdd(&count[c], 1);
}

__global__ void k_ds_scatter(const int32_t *__restrict__ cell, int64_t N, const int32_t *__restrict__ start,
                             int32_t *__restrict__ count, int32_t *__restrict__ tmp)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int c = cell[i];
    const int slot = atomicSub(&count[c], 1) - 1;                        // count returns to zero
    tmp[start[c] + slot] = (int)i;
}

__global__ void k_ds_rank(const int32_t *__restrict__ cell, const int32_t *__restrict__ tmp, int64_t N,
                          const int32_t *__restrict__ start, int32_t *__restrict__ sorted)
{
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= N) return;
    const int i = tmp[q], c = cell[i];
    const int s = start[c], e = start[c + 1];
    int r = 0;
    for (int k = s; k < e; k++) r += tmp[k] < i;
    sorted[s + r] = i;
}

// one event of one output pixel (scripts/downsample_events.py:115-122): the accumulator step of both down-samplers
// (k_ds_walk, k_stream_ingest).  pi = the event's polarity +-1, denom = fx * fy.  Returns whether the event passes.
__device__ __forceinline__ bool ds_step(float &acc, float pi, double denom)
{
    // numba: float32 array element += float64 expression  ->  sum in float64, rounded once to float32
    acc = (float)((double)acc + (double)pi * 1.0 / denom);
    const bool pass = fabsf(acc) >= 1.f;
    if (pass) acc = __fsub_rn(acc, pi);
    return pass;
}

__global__ void k_ds_walk(const int8_t *__restrict__ p, const int32_t *__restrict__ start, const int32_t *__restrict__ sorted,
                          int cells, double denom, float *__restrict__ change_map, uint8_t *__restrict__ mask)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cells) return;
    const int s = start[c], e = start[c + 1];
    if (s == e) return;
    float acc = change_map[c];
    for (int k = s; k < e; k++) {
        const int i = sorted[k];
        mask[i] = ds_step(acc, (float)p[i], denom) ? 1 : 0;
    }
    change_map[c] = acc;
}

extern "C" int dagr_downsample_events(const uint16_t *x, const uint16_t *y, const int8_t *p, int64_t N, int fx, int fy,
                                      int out_w, int out_h, float *change_map, int32_t *cell, int32_t *tmp, int32_t *sorted,
                                      int32_t *count, int32_t *start, int32_t *blocksums, uint8_t *mask, void *stream)
{
    DAGR_CHECK_ARG(change_map && count && start && blocksums, "null argument");
    DAGR_CHECK_ARG(N == 0 || (x && y && p && cell && tmp && sorted && mask), "null argument (the N-long rows may be NULL only when N = 0)");
    DAGR_CHECK_ARG(N >= 0 && N < (1ll << 31), "N must be in [0, 2^31)");
    DAGR_CHECK_ARG(fx >= 1 && fy >= 1 && out_w >= 1 && out_h >= 1, "bad down-sampling geometry: fx, fy, out_w, out_h must be >= 1");
    DAGR_CHECK_ARG((int64_t)out_w * out_h < (1ll << 31), "out_w * out_h must be < 2^31");
    if (N == 0) return DAGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int cells = out_w * out_h;
    k_ds_hist<<<dagr_div_up(N, 256), 256, 0, st>>>(x, y, N, fx, fy, out_w, out_h, cell, count);
    scan_exclusive(count, start, (int64_t)cells, blocksums, st);          // start[cells] = N
    k_ds_scatter<<<dagr_div_up(N, 256), 256, 0, st>>>(cell, N, start, count, tmp);
    k_ds_rank<<<dagr_div_up(N, 256), 256, 0, st>>>(cell, tmp, N, start, sorted);
    k_ds_walk<<<dagr_div_up(cells, 128), 128, 0, st>>>(p, start, sorted, cells, (double)fx * fy, change_map, mask);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// stable compaction of the events a mask keeps, with the output coordinates of the down-sampler
// (`(x / fx).astype("uint16")`, downsample_events.py:103-104; fx = fy = 1 leaves them unchanged)
// ------------------------------------------------------------------------------------------------
__global__ void k_mask_to_int(const uint8_t *__restrict__ mask, int64_t N, int32_t *__restrict__ flag)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) flag[i] = mask[i] ? 1 : 0;
}

__global__ void k_compact(const int32_t *__restrict__ flag, const int32_t *__restrict__ pos, int64_t N,
                          const uint16_t *__restrict__ x, const uint16_t *__restrict__ y, const int64_t *__restrict__ t,
                          const int8_t *__restrict__ p, int fx, int fy, uint16_t *__restrict__ xo, uint16_t *__restrict__ yo,
                          int64_t *__restrict__ to, int8_t *__restrict__ po)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || !flag[i]) return;
    const int j = pos[i];
    xo[j] = (uint16_t)(x[i] / fx); yo[j] = (uint16_t)(y[i] / fy); to[j] = t[i]; po[j] = p[i];
}

extern "C" int dagr_compact_events(const uint8_t *mask, int64_t N, const uint16_t *x, const uint16_t *y, const int64_t *t,
                                   const int8_t *p, int fx, int fy, int32_t *flag, int32_t *pos, int32_t *blocksums,
                                   uint16_t *xo, uint16_t *yo, int64_t *to, int8_t *po, int32_t *n_out, void *stream)
{
    DAGR_CHECK_ARG(pos && blocksums && n_out, "null argument");
    DAGR_CHECK_ARG(N == 0 || (mask && x && y && t && p && flag && xo && yo && to && po),
                   "null argument (the N-long rows may be NULL only when N = 0)");
    DAGR_CHECK_ARG(N >= 0 && N < (1ll << 31), "N must be in [0, 2^31)");
    DAGR_CHECK_ARG(fx >= 1 && fy >= 1, "fx and fy must be >= 1");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 0) { DAGR_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int32_t), st)); return DAGR_OK; }
    k_mask_to_int<<<dagr_div_up(N, 256), 256, 0, st>>>(mask, N, flag);
    scan_exclusive(flag, pos, N, blocksums, st);
    k_compact<<<dagr_div_up(N, 256), 256, 0, st>>>(flag, pos, N, x, y, t, p, fx, fy, xo, yo, to, po);
    DAGR_CUDA(cudaMemcpyAsync(n_out, pos + N, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));   // total kept
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// window slice + crop + relative time + polarity + normalise/denormalise, fused: raw events of ONE sample ->
// batch i32[M], pos i32[M,3], polarity f32[M]  (the arrays DAGR.forward derives from a formatted Batch)
// ------------------------------------------------------------------------------------------------
__global__ void k_ing_flag(const uint16_t *__restrict__ y, const int64_t *__restrict__ t, int64_t N, int H, long long t_cut,
                           int32_t *__restrict__ flag, unsigned long long *__restrict__ ilast)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool keep = false;
    if (i < N) { keep = (int)y[i] < H && t[i] < t_cut; flag[i] = keep ? 1 : 0; }
    // t[-1] of the kept events (dsec_data.py:145) is the t of the last kept event in array order, whatever the order or
    // sign of the timestamps: reduce the largest kept index (N < 2^31), -1 when nothing is kept
    int m = keep ? (int)i : -1;
    for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0 && m >= 0) atomicMax(reinterpret_cast<long long *>(ilast), (long long)m);
}

__global__ void k_ing_emit(const int32_t *__restrict__ flag, const int32_t *__restrict__ pos, int64_t N,
                           const uint16_t *__restrict__ x, const uint16_t *__restrict__ y, const int64_t *__restrict__ t,
                           const int8_t *__restrict__ p, int p_is_01, float W, float H, int T,
                           const unsigned long long *__restrict__ ilast, int b, int32_t *__restrict__ batch_o,
                           int32_t *__restrict__ pos_o, float *__restrict__ feat_o)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N || !flag[i]) return;
    const int j = pos[i];
    // data/utils.py:12-13: xy -> int16, t -> int32;  dsec_data.py:145: t = time_window + t - t[-1]
    // (a kept event exists, so ilast >= 0; the int64 sum wraps as numpy's does, and the int32 cast keeps the low bits)
    const int xi = (int)(int16_t)x[i], yi = (int)(int16_t)y[i];
    const long long tlast = t[(long long)*ilast];
    const int tr = (int)(long long)((unsigned long long)T + (unsigned long long)t[i] - (unsigned long long)tlast);
    // buffers.py:43: int / int -> fp32 true division;  ev_tgn.py:15-16: (pos * [W,H,T] + 1e-3).int()
    const float Tf = (float)T;
    const float px = __fdiv_rn((float)xi, W), py = __fdiv_rn((float)yi, H), pt = __fdiv_rn((float)tr, Tf);
    pos_o[3 * (int64_t)j] = (int)__fadd_rn(__fmul_rn(W, px), 1e-3f);
    pos_o[3 * (int64_t)j + 1] = (int)__fadd_rn(__fmul_rn(H, py), 1e-3f);
    pos_o[3 * (int64_t)j + 2] = (int)__fadd_rn(__fmul_rn(Tf, pt), 1e-3f);
    batch_o[j] = b;
    const int pv = (int)p[i];
    feat_o[j] = (float)(p_is_01 ? (int)(int8_t)(2 * pv - 1) : pv);        // dsec_data.py:146
}

extern "C" int dagr_ingest_events(const uint16_t *x, const uint16_t *y, const int64_t *t, const int8_t *p, int64_t N,
                                  int p_is_01, int W, int H, int T, int64_t t_cut, int sample, int32_t *flag, int32_t *pos,
                                  int32_t *blocksums, unsigned long long *tlast, int32_t *batch_out, int32_t *pos_out,
                                  float *feat_out, int32_t *n_out, void *stream)
{
    DAGR_CHECK_ARG(pos && blocksums && tlast && n_out, "null argument");
    DAGR_CHECK_ARG(N == 0 || (x && y && t && p && flag && batch_out && pos_out && feat_out),
                   "null argument (the N-long rows may be NULL only when N = 0)");
    DAGR_CHECK_ARG(N >= 0 && N < (1ll << 31), "N must be in [0, 2^31)");
    DAGR_CHECK_ARG(W >= 1 && H >= 1 && T >= 1, "W, H and T must be >= 1");
    cudaStream_t st = (cudaStream_t)stream;
    DAGR_CUDA(cudaMemsetAsync(tlast, 0xff, sizeof(unsigned long long), st));   // -1: no kept event yet
    if (N == 0) { DAGR_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int32_t), st)); return DAGR_OK; }
    k_ing_flag<<<dagr_div_up(N, 256), 256, 0, st>>>(y, t, N, H, (long long)t_cut, flag, tlast);
    scan_exclusive(flag, pos, N, blocksums, st);
    k_ing_emit<<<dagr_div_up(N, 256), 256, 0, st>>>(flag, pos, N, x, y, t, p, p_is_01, (float)W, (float)H, T, tlast, sample,
                                                    batch_out, pos_out, feat_out);
    DAGR_CUDA(cudaMemcpyAsync(n_out, pos + N, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));   // total kept
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// streaming ingest: the raw sensor chunks of S cameras -> the stage of dagr_stream_push[_multi], inside a captured step.
// One CTA per stream.  The chunk's events are sorted in shared memory by the key cell << 14 | arrival index (a bitonic
// sort; the keys are unique, so the order is (cell, arrival), i.e. stable), then one thread per run of equal cells walks
// its events in arrival order with ds_step, carrying that cell's accumulator in change_map.  The kept events are then
// compacted in arrival order, cropped to y / fy < crop_h, and written as (x / fx, y / fy, t, 2p - 1) rows.  At fx = fy = 1
// the walk is skipped: every event passes (0 + p reaches +-1) and the accumulator returns to 0, so the map stays 0.
// Every launch dimension is a constant of the detector; the counts are read from the raw stage on the device.
// ------------------------------------------------------------------------------------------------
#define SI_THREADS 1024
#define SI_IDX_BITS 14                          // arrival index bits of a sort key: DAGR_INGEST_MAX_RAW = 2^14
#define SI_IDX_MASK ((1u << SI_IDX_BITS) - 1u)

static_assert(DAGR_INGEST_MAX_RAW == (1 << SI_IDX_BITS), "the sort key holds the arrival index in SI_IDX_BITS bits");
static_assert((int64_t)DAGR_INGEST_MAX_CELLS << SI_IDX_BITS == (1ll << 32), "the sort key is 32 bits");

__global__ void __launch_bounds__(SI_THREADS) k_stream_ingest(const int32_t *__restrict__ raw, int S, int max_raw, int kcap, int fx,
                                                              int fy, int ow, int oh, int crop_h, float *__restrict__ change_map,
                                                              int32_t *__restrict__ stage, int max_chunk)
{
    extern __shared__ uint32_t si_key[];                                 // [kcap] sort keys
    uint8_t *keep = reinterpret_cast<uint8_t *>(si_key + kcap);          // [max_raw] the down-sampler's verdict, by arrival
    __shared__ int sm[32];
    __shared__ int tot;
    const int s = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int4 hdr = reinterpret_cast<const int4 *>(raw)[s];
    const int n = min(max(hdr.x, 0), max_raw);
    const int eo = min(max(hdr.z, 0), S * max_raw - n);                  // a bad offset cannot read past the stage
    const int2 *ev = reinterpret_cast<const int2 *>(raw + 4 * S) + eo;
    if (fx * fy > 1) {
        float *cm = change_map + (int64_t)s * ow * oh;
        const int np2 = n <= 1 ? n : 1 << (32 - __clz(n - 1));
        for (int i = tid; i < np2; i += nt) {
            uint32_t key = 0xffffffffu;                                  // padding sorts last
            if (i < n) {
                const uint32_t w = (uint32_t)ev[i].x;
                // the reference would index out of bounds; clamp as k_ds_hist does
                const int xl = min((int)(w & 0xffffu) / fx, ow - 1), yl = min((int)((w >> 16) & 0x7fffu) / fy, oh - 1);
                key = (uint32_t)(yl * ow + xl) << SI_IDX_BITS | (uint32_t)i;
            }
            si_key[i] = key;
        }
        __syncthreads();
        for (int k = 2; k <= np2; k <<= 1)
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int q = tid; q < (np2 >> 1); q += nt) {
                    const int i = 2 * q - (q & (j - 1)), l = i + j;
                    const uint32_t a = si_key[i], b = si_key[l];
                    if ((a > b) == ((i & k) == 0)) { si_key[i] = b; si_key[l] = a; }
                }
                __syncthreads();
            }
        const double denom = (double)(fx * fy);
        for (int r = tid; r < n; r += nt) {
            const uint32_t c = si_key[r] >> SI_IDX_BITS;
            if (r > 0 && (si_key[r - 1] >> SI_IDX_BITS) == c) continue;   // not the first event of its cell
            float acc = cm[c];
            int q = r;
            do {                                                         // a hot cell is walked serially, as in the reference
                const int i = (int)(si_key[q] & SI_IDX_MASK);
                keep[i] = ds_step(acc, ev[i].x < 0 ? 1.f : -1.f, denom) ? 1 : 0;
            } while (++q < n && (si_key[q] >> SI_IDX_BITS) == c);
            cm[c] = acc;
        }
    } else {
        for (int i = tid; i < n; i += nt) keep[i] = 1;
    }
    __syncthreads();
    const int obase = s * max_chunk;
    int4 *out = reinterpret_cast<int4 *>(stage + 4 * S) + obase;
    int kept = 0;
    for (int b0 = 0; b0 < n; b0 += nt) {                                 // stable compaction, nt events per round
        const int i = b0 + tid;
        int f = 0, xo = 0, yo = 0;
        int2 e = make_int2(0, 0);
        if (i < n) {
            e = ev[i];
            const uint32_t w = (uint32_t)e.x;
            xo = (int)(w & 0xffffu) / fx;                                // (x / fx).astype(uint16), downsample_events.py:103
            yo = (int)((w >> 16) & 0x7fffu) / fy;
            f = keep[i] && yo < crop_h;                                  // crop, dsec_data.py:142-143
        }
        const int off = block_exclusive_scan(f, &tot, sm);
        if (f) out[kept + off] = make_int4(xo, yo, e.y, e.x < 0 ? 1 : -1);
        kept += tot;
    }
    if (tid == 0) reinterpret_cast<int4 *>(stage)[s] = make_int4(kept, hdr.y, obase, hdr.w);
}

extern "C" int dagr_stream_ingest(const int32_t *raw_stage, int streams, int max_raw, int fx, int fy, int out_w, int out_h, int crop_h,
                                  float *change_map, int32_t *stage, int max_chunk, void *stream)
{
    DAGR_CHECK_ARG(raw_stage && change_map && stage, "null argument");
    DAGR_CHECK_ARG(streams >= 1 && streams <= 127, "streams must be in [1, 127]");
    DAGR_CHECK_ARG(fx >= 1 && fy >= 1, "fx and fy must be >= 1");
    DAGR_CHECK_ARG(out_w >= 1 && out_h >= 1 && (int64_t)out_w * fx <= (1 << 16) && (int64_t)out_h * fy <= (1 << 15),
                   "bad geometry: the raw record holds x in 16 bits and y in 15 bits (out_w * fx <= 65536, out_h * fy <= 32768)");
    DAGR_CHECK_ARG(fx * fy == 1 || (int64_t)out_w * out_h <= DAGR_INGEST_MAX_CELLS,
                   "more than 2^18 output cells: the sort key is cell << 14 | arrival index in 32 bits");
    DAGR_CHECK_ARG(crop_h >= 1 && crop_h <= out_h, "crop_h must be in [1, out_h]");
    DAGR_CHECK_ARG(max_raw >= 1 && max_raw <= DAGR_INGEST_MAX_RAW, "max_raw must be in [1, 16384] (shared-memory sort)");
    DAGR_CHECK_ARG(max_raw <= max_chunk, "max_raw must be <= max_chunk (a stream's kept events fill its stage slot)");
    int kcap = 1;
    while (kcap < max_raw) kcap <<= 1;
    const size_t smem = (size_t)kcap * sizeof(uint32_t) + (size_t)(max_raw + 15) / 16 * 16;
    DAGR_CUDA(dagr_allow_smem(k_stream_ingest, smem));
    k_stream_ingest<<<streams, SI_THREADS, smem, (cudaStream_t)stream>>>(raw_stage, streams, max_raw, kcap, fx, fy, out_w, out_h, crop_h,
                                                                         change_map, stage, max_chunk);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// windows of one recording (dagr_b200.sequence): the live-window rule of the rings applied to a time-sorted recording,
// then a block of G windows gathered as the G samples of one batched forward.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int lower_bound_i64(const int64_t *__restrict__ t, int n, long long v)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
        if (__ldg(t + mid) < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void k_window_bounds(const int64_t *__restrict__ t, int n, const int64_t *__restrict__ t_begin,
                                const int64_t *__restrict__ t_end, int64_t Q, int32_t *__restrict__ begin, int32_t *__restrict__ end)
{
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= Q) return;
    begin[q] = lower_bound_i64(t, n, (long long)t_begin[q]);
    end[q] = lower_bound_i64(t, n, (long long)t_end[q]);
}

extern "C" int dagr_window_bounds(const int64_t *t, int64_t N, const int64_t *t_begin, const int64_t *t_end, int64_t Q,
                                  int32_t *begin, int32_t *end, void *stream)
{
    DAGR_CHECK_ARG(N == 0 || t, "null t (it may be NULL only when N = 0)");
    DAGR_CHECK_ARG(Q == 0 || (t_begin && t_end && begin && end), "null argument (the Q-long rows may be NULL only when Q = 0)");
    DAGR_CHECK_ARG(N >= 0 && N < (1ll << 31), "N must be in [0, 2^31)");
    DAGR_CHECK_ARG(Q >= 0 && Q < (1ll << 31), "Q must be in [0, 2^31)");
    if (Q == 0) return DAGR_OK;
    k_window_bounds<<<dagr_div_up(Q, 256), 256, 0, (cudaStream_t)stream>>>(t, (int)N, t_begin, t_end, Q, begin, end);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// One CTA per WG_ROWS consecutive output rows.  Every CTA scans the G window sizes itself (G <= 255: one value per thread;
// two int block scans of the high and low bits give the exact 64-bit offsets of any begin / end), then each thread finds
// the window of its row by a binary search over the offsets in shared memory and copies one event: consecutive threads
// read consecutive events of one window and write consecutive rows, and no two CTAs write the same row, so there are no
// atomics.
#define WG_THREADS 256
#define WG_ROWS (WG_THREADS * 4)

__global__ void __launch_bounds__(WG_THREADS) k_window_gather(const uint16_t *__restrict__ x, const uint16_t *__restrict__ y,
                                                               const int64_t *__restrict__ t, const int8_t *__restrict__ p,
                                                               const int32_t *__restrict__ begin, const int32_t *__restrict__ end,
                                                               int G, long long t_base, int p_is_01, int total,
                                                               int32_t *__restrict__ batch_o, int32_t *__restrict__ pos_o,
                                                               float *__restrict__ feat_o, int64_t *__restrict__ offsets)
{
    __shared__ long long off[WG_THREADS];
    __shared__ int src[WG_THREADS];
    __shared__ int sm[32];
    __shared__ int tot_hi, tot_lo;
    const int tid = threadIdx.x;
    int b = 0, n = 0;
    if (tid < G) { b = begin[tid]; n = max(end[tid] - b, 0); }
    const int o_hi = block_exclusive_scan(n >> 12, &tot_hi, sm);         // <= 2^19 per window: no int overflow
    const int o_lo = block_exclusive_scan(n & 4095, &tot_lo, sm);
    off[tid] = (long long)o_hi * 4096 + o_lo;
    src[tid] = b;
    __syncthreads();
    const long long tot = (long long)tot_hi * 4096 + tot_lo;
    if (blockIdx.x == 0 && tid <= G) offsets[tid] = tid < G ? off[tid] : tot;
    const int rows = (int)min(tot, (long long)total);                    // the caller's rows bound every write
    for (int r = blockIdx.x * WG_ROWS + tid; r < min(rows, (int)(blockIdx.x + 1) * WG_ROWS); r += WG_THREADS) {
        int lo = 0, hi = G - 1;                                          // the last window w with off[w] <= r
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (off[mid] <= r) lo = mid;
            else hi = mid - 1;
        }
        const int64_t i = (int64_t)src[lo] + (r - off[lo]);
        batch_o[r] = lo;
        pos_o[3 * (int64_t)r] = (int)__ldg(x + i);
        pos_o[3 * (int64_t)r + 1] = (int)__ldg(y + i);
        pos_o[3 * (int64_t)r + 2] = (int)((long long)__ldg(t + i) - t_base);
        const int pv = (int)__ldg(p + i);
        feat_o[r] = (float)(p_is_01 ? 2 * pv - 1 : pv);
    }
}

extern "C" int dagr_window_gather(const uint16_t *x, const uint16_t *y, const int64_t *t, const int8_t *p, int64_t N,
                                  const int32_t *begin, const int32_t *end, int G, int64_t t_base, int p_is_01, int64_t total,
                                  int32_t *batch_out, int32_t *pos_out, float *feat_out, int64_t *offsets, void *stream)
{
    DAGR_CHECK_ARG(begin && end && offsets, "null argument");
    DAGR_CHECK_ARG(N == 0 || (x && y && t && p), "null argument (the N-long rows may be NULL only when N = 0)");
    DAGR_CHECK_ARG(total == 0 || (batch_out && pos_out && feat_out), "null argument (the output rows may be NULL only when total = 0)");
    DAGR_CHECK_ARG(N >= 0 && N < (1ll << 31), "N must be in [0, 2^31)");
    DAGR_CHECK_ARG(G >= 1 && G <= 255, "G must be in [1, 255] (the windows of a block are the samples of one forward)");
    DAGR_CHECK_ARG(total >= 0 && total < (1ll << 24), "the block total must be in [0, 2^24) (sorted positions are packed in 24 bits)");
    const int ctas = total > 0 ? dagr_div_up(total, WG_ROWS) : 1;
    k_window_gather<<<ctas, WG_THREADS, 0, (cudaStream_t)stream>>>(x, y, t, p, begin, end, G, (long long)t_base, p_is_01, (int)total,
                                                                  batch_out, pos_out, feat_out, offsets);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// camera frames (dsec_data.py:149-154): crop to scale * H rows, cv2.resize(INTER_CUBIC) by the integer factor `scale`,
// HWC -> CHW, in one pass.  At an integer factor the cubic is integer arithmetic (oracle/ref_frame.py): the source
// coordinate of output pixel d is (d + 0.5) * s - 0.5.  Odd s: fraction 0, the output is source pixel s * d + (s - 1) / 2.
// Even s: sx = s * d + s / 2 - 1, fraction 0.5, taps sx - 1 .. sx + 2 clamped to the cropped frame with weights
// [-3, 19, 19, -3] / 32 per axis; the 16-tap sum (units of 1/1024) is rounded half to even and saturated.  No floating
// point, so no contraction or summation order can change a bit.  The f32 form maps the byte through `lut` (the caller's
// torch u8 -> f32 / 255.0 table, so the bits are those of `.float() / 255.0` on the device).
// One thread per output pixel, all three channels.  The taps are read straight from global memory: at s = 2 neighbouring
// threads share half their taps and the L1 serves the repeats; at s >= 4 no tap is shared.  A 640x480 frame is 0.9 MB.
// ------------------------------------------------------------------------------------------------
#define FP_THREADS 128

__device__ __forceinline__ int fp_round(int v)                          // round(v / 1024) half to even, saturated to [0, 255]
{
    int q = v >> 10;                                                     // floor
    const int r = v & 1023;
    q += (r > 512) | ((r == 512) & (q & 1));
    return min(max(q, 0), 255);
}

template <bool F32>
__global__ void __launch_bounds__(FP_THREADS) k_frame_preprocess(const uint8_t *__restrict__ src, int sh, int sw, int s, int H, int W,
                                                                 uint8_t *__restrict__ out_u8, float *__restrict__ out_f32,
                                                                 const float *__restrict__ lut)
{
    const int x = blockIdx.x * FP_THREADS + threadIdx.x, y = blockIdx.y, f = blockIdx.z;
    if (x >= W) return;
    const uint8_t *img = src + (int64_t)f * sh * sw * 3;
    int v[3];
    if (s & 1) {
        const uint8_t *px = img + ((int64_t)(s * y + (s - 1) / 2) * sw + s * x + (s - 1) / 2) * 3;
        v[0] = __ldg(px); v[1] = __ldg(px + 1); v[2] = __ldg(px + 2);
    } else {
        const int wt[4] = {-3, 19, 19, -3};
        const int ch = s * H;                                            // the cropped frame's rows: the border cv2 replicates
        const int sy = s * y + s / 2 - 1, sx = s * x + s / 2 - 1;
        int cx[4];
#pragma unroll
        for (int k = 0; k < 4; k++) cx[k] = 3 * min(max(sx - 1 + k, 0), sw - 1);
        int acc[3] = {0, 0, 0};
#pragma unroll
        for (int ky = 0; ky < 4; ky++) {
            const uint8_t *row = img + (int64_t)min(max(sy - 1 + ky, 0), ch - 1) * sw * 3;
            int hs[3] = {0, 0, 0};
#pragma unroll
            for (int kx = 0; kx < 4; kx++)
#pragma unroll
                for (int c = 0; c < 3; c++) hs[c] += wt[kx] * (int)__ldg(row + cx[kx] + c);
#pragma unroll
            for (int c = 0; c < 3; c++) acc[c] += wt[ky] * hs[c];
        }
#pragma unroll
        for (int c = 0; c < 3; c++) v[c] = fp_round(acc[c]);
    }
    const int64_t plane = (int64_t)H * W, o = (int64_t)f * 3 * plane + (int64_t)y * W + x;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        if (F32) out_f32[o + c * plane] = __ldg(lut + v[c]);
        else out_u8[o + c * plane] = (uint8_t)v[c];
    }
}

extern "C" int dagr_frame_preprocess(const uint8_t *frames, int nframes, int src_h, int src_w, int scale, int out_h, int out_w,
                                     uint8_t *out_u8, float *out_f32, const float *lut, void *stream)
{
    DAGR_CHECK_ARG(frames, "null frames");
    DAGR_CHECK_ARG((out_u8 != nullptr) != (out_f32 != nullptr), "exactly one of out_u8 / out_f32 must be given");
    DAGR_CHECK_ARG(!out_f32 || lut, "null lut: the f32 output needs the 256-entry u8 -> f32 table");
    DAGR_CHECK_ARG(nframes >= 1 && nframes <= 65535, "nframes must be in [1, 65535]");
    DAGR_CHECK_ARG(out_w >= 1 && out_h >= 1 && out_h <= 65535, "out_w >= 1 and 1 <= out_h <= 65535");
    DAGR_CHECK_ARG(scale >= 1, "scale must be >= 1");
    DAGR_CHECK_ARG((int64_t)src_w == (int64_t)scale * out_w, "src_w must equal scale * out_w (integer factors only)");
    DAGR_CHECK_ARG((int64_t)src_h >= (int64_t)scale * out_h, "src_h must be >= scale * out_h (the crop keeps scale * out_h rows)");
    DAGR_CHECK_ARG((int64_t)src_h * src_w * 3 < (1ll << 31), "a frame must hold fewer than 2^31 bytes");
    const dim3 grid(dagr_div_up(out_w, FP_THREADS), out_h, nframes);
    if (out_f32)
        k_frame_preprocess<true><<<grid, FP_THREADS, 0, (cudaStream_t)stream>>>(frames, src_h, src_w, scale, out_h, out_w, nullptr, out_f32, lut);
    else
        k_frame_preprocess<false><<<grid, FP_THREADS, 0, (cudaStream_t)stream>>>(frames, src_h, src_w, scale, out_h, out_w, out_u8, nullptr,
                                                                                 nullptr);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}
