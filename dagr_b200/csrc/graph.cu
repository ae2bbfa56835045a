// graph.cu -- causal spatio-temporal radius graph over (x,y,t) events, sm_90a.
//
// Replaces the reference's [B,Q,H,W] FIFO (src/dagr/graph/ev_graph.cu:169-212) + spiral probe
// (ev_graph.cu:15-80, spiral.h) with:
//   1. a counting sort of the batch by a CELL-MAJOR pixel key (pool1 voxel, then pixel inside the
//      voxel, then arrival order).  A pixel's FIFO column == the tail of its bin read backwards;
//      a pool1 voxel's members == one contiguous range, which is what lets the event-level convs
//      and pool1 run as streaming, coalesced passes with warp-segmented reductions.
//   2. a probe that walks the same spiral over bins and writes a column-major ELL adjacency (slot q
//      of node p at [q*N + p]) in probe order, so that every later pass reads it fully coalesced.
//      It runs per pool1 voxel on staged records, fused with conv_a (build_l1.cu).
#include "common.cuh"

#define SCAN_THREADS 256
#define SCAN_ITEMS 8
#define SCAN_TILE (SCAN_THREADS * SCAN_ITEMS)

extern "C" int64_t dagr_scan_blocks(int64_t n) { return (n + SCAN_TILE - 1) / SCAN_TILE; }

// ------------------------------------------------------------------------------------------------
// exclusive scan (int32), three small kernels.  out may alias in.  (block_exclusive_scan: common.cuh)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_reduce(const int *__restrict__ in, int64_t n, int *__restrict__ blocksums)
{
    __shared__ int sm[32];
    __shared__ int tot;
    int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
    int s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { int64_t i = base + k; if (i < n) s += in[i]; }
    block_exclusive_scan(s, &tot, sm);
    if (threadIdx.x == 0) blocksums[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_blocksums(int *__restrict__ blocksums, int64_t nb)
{
    // single block, sequential over chunks with a running carry; writes exclusive prefix in place and
    // the grand total at blocksums[nb]
    __shared__ int sm[32];
    __shared__ int tot;
    int carry = 0;
    for (int64_t c = 0; c < nb; c += SCAN_THREADS) {
        int64_t i = c + threadIdx.x;
        int v = (i < nb) ? blocksums[i] : 0;
        int ex = block_exclusive_scan(v, &tot, sm);
        if (i < nb) blocksums[i] = ex + carry;
        carry += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) blocksums[nb] = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_apply(const int *__restrict__ in, int *__restrict__ out, int64_t n,
                                                             const int *__restrict__ blocksums, int64_t nb)
{
    __shared__ int sm[32];
    __shared__ int tot;
    int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS];
    int s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { int64_t i = base + k; v[k] = (i < n) ? in[i] : 0; s += v[k]; }
    int ex = block_exclusive_scan(s, &tot, sm) + blocksums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { int64_t i = base + k; if (i < n) out[i] = ex; ex += v[k]; }
    if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = blocksums[nb];   // total
}

// out[0..n-1] = exclusive prefix of in, out[n] = total.  blocksums: dagr_scan_blocks(n)+1 ints.
int scan_exclusive(const int *in, int *out, int64_t n, int *blocksums, cudaStream_t st)
{
    int64_t nb = dagr_scan_blocks(n);
    if (nb == 0) nb = 1;
    k_scan_reduce<<<(unsigned)nb, SCAN_THREADS, 0, st>>>(in, n, blocksums);
    k_scan_blocksums<<<1, SCAN_THREADS, 0, st>>>(blocksums, nb);
    k_scan_apply<<<(unsigned)nb, SCAN_THREADS, 0, st>>>(in, out, n, blocksums, nb);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// a1' denormalize_pos
// ------------------------------------------------------------------------------------------------
__global__ void k_denorm(const float *__restrict__ pos, int64_t n3, float W, float H, float T, int32_t *__restrict__ out)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n3) return;
    int d = (int)(i % 3);
    float s = d == 0 ? W : (d == 1 ? H : T);
    // (denorm * pos + 1e-3).int(): separate fp32 multiply and add, then truncation (ev_tgn.py:15-16)
    out[i] = (int)__fadd_rn(__fmul_rn(s, pos[i]), 1e-3f);
}

extern "C" int dagr_denormalize_pos(const float *pos, int64_t N, int W, int H, int T, int32_t *pos_i32, void *stream)
{
    if (N <= 0) return DAGR_OK;
    int64_t n3 = 3 * N;
    k_denorm<<<dagr_div_up(n3, 256), 256, 0, (cudaStream_t)stream>>>(pos, n3, (float)W, (float)H, (float)T, pos_i32);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// The whole input conversion of DAGR.forward in one pass: denormalize_pos (above), batch int64 -> int32 (ev_tgn.py:57
// passes events.batch.int()) and the polarity column of x as a dense fp32 vector.
__global__ void k_prepare_events(const float *__restrict__ pos, const int64_t *__restrict__ batch64, const float *__restrict__ x, int ldx,
                                 int64_t N, float W, float H, float T, int32_t *__restrict__ pos_i, int32_t *__restrict__ batch_i,
                                 float *__restrict__ feat)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    pos_i[3 * i + 0] = (int)__fadd_rn(__fmul_rn(W, pos[3 * i + 0]), 1e-3f);
    pos_i[3 * i + 1] = (int)__fadd_rn(__fmul_rn(H, pos[3 * i + 1]), 1e-3f);
    pos_i[3 * i + 2] = (int)__fadd_rn(__fmul_rn(T, pos[3 * i + 2]), 1e-3f);
    batch_i[i] = (int32_t)batch64[i];
    feat[i] = x[i * ldx];
}

extern "C" int dagr_prepare_events(const float *pos, const int64_t *batch, const float *x, int ldx, int64_t N, int W, int H, int T,
                                   int32_t *pos_i32, int32_t *batch_i32, float *feat, void *stream)
{
    if (N <= 0) return DAGR_OK;
    DAGR_CHECK_ARG(pos && batch && x && pos_i32 && batch_i32 && feat && ldx >= 1, "bad argument");
    k_prepare_events<<<dagr_div_up(N, 256), 256, 0, (cudaStream_t)stream>>>(pos, batch, x, ldx, N, (float)W, (float)H, (float)T, pos_i32,
                                                                          batch_i32, feat);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// sort
// ------------------------------------------------------------------------------------------------
// Streaming form (dagr_graph_sort_ring[s]): the events live in S ring buffers of `mask + 1` slots each (ring s owns
// slots [s*(mask+1), (s+1)*(mask+1))) and the live windows are described by a DEVICE control block (dagr_stream_push
// [_multi] below).  The windows are read in one compact, stream-major arrival order c < total: stream s holds
// c in [off_s, off_s + live_s), and its i-th live event (i = c - off_s) is slot s*(mask+1) + ((head_s + i) & mask).  The
// launch covers all S*(mask+1) slots -- so the grid does not depend on the live counts and the step can be replayed as a
// CUDA graph.  The single-ring control block (i32[8], no offsets, no total block) is the S = 1 case: off_0 = 0 and the
// total is its live count.  ctl == nullptr is the plain (non-ring) sort over N events.
struct RingAt {
    int64_t slot;      // ring slot of the event
    int i;             // its index inside its stream's live window
};

__device__ __forceinline__ int64_t ring_total(const int32_t *ctl, int S, int64_t N)
{
    if (ctl == nullptr) return N;
    return S == 1 ? (int64_t)ctl[1] : (int64_t)ctl[DAGR_RING_CTL * S];
}

__device__ __forceinline__ RingAt ring_at(const int32_t *ctl, int S, int mask, int c)
{
    if (ctl == nullptr) return RingAt{(int64_t)c, c};
    int s = 0;
    if (S > 1) {                                                        // last stream whose window starts at or before c
        int lo = 0, hi = S - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (__ldg(ctl + DAGR_RING_CTL * mid + 6) <= c) lo = mid; else hi = mid - 1;
        }
        s = lo;
    }
    const int32_t *cs = ctl + DAGR_RING_CTL * s;
    const int i = S > 1 ? c - __ldg(cs + 6) : c;
    return RingAt{(int64_t)s * (mask + 1) + ((__ldg(cs) + i) & mask), i};
}

__global__ void k_keys_hist(dagr_geom_t g, const int32_t *__restrict__ batch, const int32_t *__restrict__ pos, int64_t N,
                            int32_t *__restrict__ key, int32_t *__restrict__ count, int32_t *__restrict__ flags,
                            const int32_t *__restrict__ ctl, int mask, int S)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ring_total(ctl, S, N)) return;
    const RingAt at = ring_at(ctl, S, mask, (int)i);
    const int64_t si = at.slot;
    int x = pos[3 * si], y = pos[3 * si + 1], b = batch[si];
    // out-of-range events are clamped into the grid (the reference would index out of bounds)
    x = min(max(x, 0), g.W - 1); y = min(max(y, 0), g.H - 1); b = min(max(b, 0), g.B - 1);
    // time-order proof for the build kernel's time-bucket pruning (SURVEY 8b): flags[0] = 1 unless the (clamped) samples
    // come as ascending contiguous runs, each time-sorted in arrival order.  Comparing every event with its predecessor
    // proves exactly that; interleaved samples count as unproven.  Without the proof the build does not prune (results
    // stay exact, only slower).  In ring mode the compact order is stream-major with ascending samples by construction,
    // and the predecessor of a stream's first live event is not compared.
    if (flags != nullptr && at.i > 0) {
        const int64_t sp = ctl != nullptr ? (si & ~(int64_t)mask) | ((si - 1) & mask) : si - 1;
        const int pb = min(max(batch[sp], 0), g.B - 1);
        if (pb > b || (pb == b && pos[3 * sp + 2] > pos[3 * si + 2])) flags[0] = 1;
    }
    int k = b * (g.ny1 * g.nx1 * g.CP) + __ldg(g.ykey + y) + __ldg(g.xkey + x);
    key[i] = k;
    atomicAdd(count + k, 1);
}

__global__ void k_scatter(const int32_t *__restrict__ key, int64_t N, const int32_t *__restrict__ start,
                          int32_t *__restrict__ count, int32_t *__restrict__ tmp, const int32_t *__restrict__ ctl, int S)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ring_total(ctl, S, N)) return;
    int k = key[i];
    int slot = atomicSub(count + k, 1) - 1;          // leaves count[] all-zero again
    tmp[start[k] + slot] = (int)i;
}

// order each bin by arrival index (stable sort of graph/utils.py:10) and emit the sorted records
__global__ void k_rank_emit(dagr_geom_t g, const int32_t *__restrict__ key, const int32_t *__restrict__ tmp, int64_t N,
                            const int32_t *__restrict__ start, const int32_t *__restrict__ batch,
                            const int32_t *__restrict__ pos, const float *__restrict__ feat,
                            int32_t *__restrict__ perm, int2 *__restrict__ ti, uint32_t *__restrict__ xyb,
                            float *__restrict__ feat_s, const int32_t *__restrict__ ctl, int mask, int S)
{
    int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ring_total(ctl, S, N)) return;
    int i = tmp[j];
    int k = key[i];
    int s = start[k], e = start[k + 1];
    int rank = 0;
    for (int q = s; q < e; q++) rank += (tmp[q] < i);
    int p = s + rank;
    const int64_t si = ring_at(ctl, S, mask, i).slot;
    int x = pos[3 * si], y = pos[3 * si + 1], t = pos[3 * si + 2], b = batch[si];
    x = min(max(x, 0), g.W - 1); y = min(max(y, 0), g.H - 1); b = min(max(b, 0), g.B - 1);
    perm[p] = i;
    ti[p] = make_int2(t, i);
    xyb[p] = (uint32_t)x | ((uint32_t)y << 12) | ((uint32_t)b << 24);
    feat_s[p] = feat[si];
}

// N = number of events (plain sort) or S * capacity (ring sort: the launches cover every slot of the S rings)
static int graph_sort_impl(const dagr_geom_t *g, const int32_t *batch, const int32_t *pos, const float *feat,
                           int64_t N, const int32_t *ctl, int mask, int S, int32_t *key, int32_t *tmp, int32_t *count,
                           int32_t *blocksums, int32_t *start, int32_t *perm, int32_t *ti, uint32_t *xyb, float *feat_s,
                           int32_t *flags, void *stream)
{
    DAGR_CHECK_ARG(g && g->W <= 4096 && g->H <= 4096 && g->B <= 256, "geometry out of range (W,H<=4096, B<=256)");
    const int64_t nk = (int64_t)g->B * g->ny1 * g->nx1 * g->CP;      // the keys and the count / start tables are int32
    DAGR_CHECK_ARG(nk < (1ll << 31) && g->NK == nk, "geometry out of range (NK = B*ny1*nx1*CP must be < 2^31: 32-bit sort key)");
    DAGR_CHECK_ARG(N >= 0 && N < (1ll << 31), "N out of range");
    cudaStream_t st = (cudaStream_t)stream;
    if (N > 0) {
        k_keys_hist<<<dagr_div_up(N, 256), 256, 0, st>>>(*g, batch, pos, N, key, count, flags, ctl, mask, S);
        DAGR_CHECK_LAUNCH();
    }
    scan_exclusive(count, start, g->NK, blocksums, st);      // start[NK] = N
    DAGR_CHECK_LAUNCH();
    if (N > 0) {
        k_scatter<<<dagr_div_up(N, 256), 256, 0, st>>>(key, N, start, count, tmp, ctl, S);
        k_rank_emit<<<dagr_div_up(N, 256), 256, 0, st>>>(*g, key, tmp, N, start, batch, pos, feat, perm,
                                                         (int2 *)ti, xyb, feat_s, ctl, mask, S);
        DAGR_CHECK_LAUNCH();
    }
    return DAGR_OK;
}

extern "C" int dagr_graph_sort(const dagr_geom_t *g, const int32_t *batch, const int32_t *pos, const float *feat,
                               int64_t N, int32_t *key, int32_t *tmp, int32_t *count, int32_t *blocksums,
                               int32_t *start, int32_t *perm, int32_t *ti, uint32_t *xyb, float *feat_s,
                               int32_t *flags, void *stream)
{
    return graph_sort_impl(g, batch, pos, feat, N, nullptr, 0, 1, key, tmp, count, blocksums, start, perm, ti, xyb, feat_s, flags,
                           stream);
}

// the limits of S rings of `capacity` slots (include/dagr_b200.h, streaming block).  The push advances all rings in one
// CTA of up to RING_MAX_STREAMS threads; with the default capacity of 2^17, S * capacity < 2^24 allows 127 streams too.
#define RING_MAX_STREAMS 128
static int check_rings(const char *who, int64_t capacity, int streams, int max_chunk)
{
    const char *msg = nullptr;
    if (streams < 1 || streams >= RING_MAX_STREAMS) msg = "streams must be in [1, 127]";
    else if (capacity <= 0 || (capacity & (capacity - 1)) != 0) msg = "ring capacity must be a power of two";
    else if ((int64_t)streams * capacity >= (1ll << 24)) msg = "streams * capacity must be < 2^24 (sorted positions are packed in 24 bits)";
    else if (max_chunk <= 0 || max_chunk > capacity) msg = "max_chunk must be in [1, capacity]";
    if (msg == nullptr) return DAGR_OK;
    dagr_set_error("%s: %s", who, msg);
    return DAGR_E_ARG;
}

extern "C" int dagr_graph_sort_ring(const dagr_geom_t *g, const int32_t *batch, const int32_t *pos, const float *feat,
                                    int64_t capacity, const int32_t *ctl, int32_t *key, int32_t *tmp, int32_t *count,
                                    int32_t *blocksums, int32_t *start, int32_t *perm, int32_t *ti, uint32_t *xyb, float *feat_s,
                                    int32_t *flags, void *stream)
{
    DAGR_CHECK_ARG(ctl != nullptr && capacity > 0 && (capacity & (capacity - 1)) == 0, "ring capacity must be a power of two");
    return graph_sort_impl(g, batch, pos, feat, capacity, ctl, (int)(capacity - 1), 1, key, tmp, count, blocksums, start, perm, ti,
                           xyb, feat_s, flags, stream);
}

extern "C" int dagr_graph_sort_rings(const dagr_geom_t *g, const int32_t *batch, const int32_t *pos, const float *feat,
                                     int64_t capacity, int streams, const int32_t *ctl, int32_t *key, int32_t *tmp, int32_t *count,
                                     int32_t *blocksums, int32_t *start, int32_t *perm, int32_t *ti, uint32_t *xyb, float *feat_s,
                                     int32_t *flags, void *stream)
{
    DAGR_CHECK_ARG(g && batch && pos && feat && ctl && key && tmp && count && blocksums && start && perm && ti && xyb && feat_s,
                   "null argument");
    const int rc = check_rings(__func__, capacity, streams, 1);
    if (rc != DAGR_OK) return rc;
    DAGR_CHECK_ARG(streams == g->B, "streams must equal the geometry's batch size B (stream s is sample s)");
    return graph_sort_impl(g, batch, pos, feat, (int64_t)streams * capacity, ctl, (int)(capacity - 1), streams, key, tmp, count,
                           blocksums, start, perm, ti, xyb, feat_s, flags, stream);
}

// ------------------------------------------------------------------------------------------------
// streaming windows (SURVEY 8d config 5; the idea of the min_index watermark of ev_graph.cu:62 / ev_graph.py:121-136):
// the live events of each of S streams sit time-sorted in their own ring; a step evicts each window's prefix older than
// its t_cut (O(log n) search, no data movement) and appends the stream's new chunk behind its tail.
//   ctl   i32[S+1][8] : block s = [0] head slot (inside ring s), [1] live count, [2] evicted by the last step, [3] appended
//                       by the last step, [4] sticky overflow flag (chunk did not fit: oldest events were dropped beyond
//                       t_cut), [5] kept count, [6] offset of the window in the stream-major order (exclusive scan of
//                       the live counts); block S = [0] total live count
//   stage i32[4*S + 4*S*max_chunk] : header [S][4] = {n_new, t_cut, event offset, 0}, then (x, y, t, polarity +-1) of
//                       all streams back to back; stream s's events start at event `offset`
// The single-stream form (dagr_stream_push) is S = 1 with a control block of one i32[8] and no total block: its stage
// {n_new, t_cut, 0, 0, events} is the S = 1 stage, and ctl[6] is written as 0.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(RING_MAX_STREAMS) k_stream_advance(int32_t *__restrict__ ctl, const int32_t *__restrict__ stage,
                                                                    const int32_t *__restrict__ pos, int mask, int max_chunk, int S,
                                                                    int32_t *__restrict__ total)
{
    __shared__ int sm[32];
    __shared__ int tot;
    const int s = threadIdx.x;
    int live = 0;
    if (s < S) {
        int32_t *c = ctl + DAGR_RING_CTL * s;
        const int head = c[0], n = c[1];
        const int n_new = min(max(stage[4 * s], 0), max_chunk), t_cut = stage[4 * s + 1];
        const int64_t base = (int64_t)s * (mask + 1);
        int lo = 0, hi = n;
        while (lo < hi) {                                               // first live event with t >= t_cut
            const int mid = (lo + hi) >> 1;
            if (pos[3 * (base + ((head + mid) & mask)) + 2] < t_cut) lo = mid + 1; else hi = mid;
        }
        int shift = lo;
        const int cap = mask + 1;
        if (n - shift + n_new > cap) { shift = n + n_new - cap; c[4] = 1; }
        c[0] = (head + shift) & mask;
        c[5] = n - shift;
        c[1] = live = n - shift + n_new;
        c[2] = shift;
        c[3] = n_new;
    }
    const int off = block_exclusive_scan(live, &tot, sm);
    if (s < S) ctl[DAGR_RING_CTL * s + 6] = off;
    if (total != nullptr && s == 0) *total = tot;
}

__global__ void k_stream_append(const int32_t *__restrict__ ctl, const int32_t *__restrict__ stage, int32_t *__restrict__ batch,
                                int32_t *__restrict__ pos, float *__restrict__ feat, int mask, int max_chunk, int sample, int S)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;     // gridDim.y = S
    const int32_t *c = ctl + DAGR_RING_CTL * s;
    const int n_new = c[3];
    if (j >= n_new) return;
    const int64_t slot = (int64_t)s * (mask + 1) + ((c[0] + c[5] + j) & mask);
    const int eo = min(max(stage[4 * s + 2], 0), S * max_chunk - n_new);     // a bad offset cannot read past the stage
    const int4 e = reinterpret_cast<const int4 *>(stage + 4 * S)[eo + j];
    pos[3 * slot] = e.x; pos[3 * slot + 1] = e.y; pos[3 * slot + 2] = e.z;
    feat[slot] = (float)e.w;
    batch[slot] = S > 1 ? s : sample;
}

static void stream_push_launch(int32_t *ctl, const int32_t *stage, int32_t *batch, int32_t *pos, float *feat, int64_t capacity,
                               int S, int max_chunk, int sample, int32_t *total, cudaStream_t st)
{
    k_stream_advance<<<1, (S + 31) / 32 * 32, 0, st>>>(ctl, stage, pos, (int)(capacity - 1), max_chunk, S, total);
    k_stream_append<<<dim3(dagr_div_up(max_chunk, 256), S), 256, 0, st>>>(ctl, stage, batch, pos, feat, (int)(capacity - 1), max_chunk,
                                                                          sample, S);
}

extern "C" int dagr_stream_push(int32_t *ctl, const int32_t *stage, int32_t *batch, int32_t *pos, float *feat, int64_t capacity,
                                int max_chunk, int sample, void *stream)
{
    DAGR_CHECK_ARG(ctl && stage && batch && pos && feat, "null argument");
    DAGR_CHECK_ARG(capacity > 0 && (capacity & (capacity - 1)) == 0 && max_chunk > 0 && max_chunk <= capacity,
                   "ring capacity must be a power of two >= max_chunk");
    stream_push_launch(ctl, stage, batch, pos, feat, capacity, 1, max_chunk, sample, nullptr, (cudaStream_t)stream);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

extern "C" int dagr_stream_push_multi(int32_t *ctl, const int32_t *stage, int32_t *batch, int32_t *pos, float *feat, int64_t capacity,
                                      int streams, int max_chunk, void *stream)
{
    DAGR_CHECK_ARG(ctl && stage && batch && pos && feat, "null argument");
    const int rc = check_rings(__func__, capacity, streams, max_chunk);
    if (rc != DAGR_OK) return rc;
    stream_push_launch(ctl, stage, batch, pos, feat, capacity, streams, max_chunk, 0, ctl + DAGR_RING_CTL * streams,
                       (cudaStream_t)stream);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

// ------------------------------------------------------------------------------------------------
// export to the reference's edge_index layout (tests / API compatibility, not on the hot path)
// ------------------------------------------------------------------------------------------------
__global__ void k_inv_deg(int64_t N, const int32_t *__restrict__ perm, const int32_t *__restrict__ nbr,
                          int32_t *__restrict__ inv, int32_t *__restrict__ degA)
{
    int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    int i = perm[p];
    inv[i] = (int)p;
    degA[i] = nbr[(int64_t)(DAGR_ELL - 1) * N + p] + 1;       // + self loop
}

__global__ void k_export(int64_t N, const int32_t *__restrict__ inv, const int2 *__restrict__ ti,
                         const int32_t *__restrict__ nbr, const int32_t *__restrict__ rowptr,
                         int64_t *__restrict__ esrc, int64_t *__restrict__ edst, int64_t cap)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    int p = inv[i];
    int64_t o = rowptr[i];
    int n = nbr[(int64_t)(DAGR_ELL - 1) * N + p];
    if (o + n + 1 > cap) return;
    esrc[o] = i; edst[o] = i;                               // self loop first (ev_graph.cu:44-46)
    for (int q = 0; q < n; q++) {
        int j = nbr[(int64_t)q * N + p];
        esrc[o + 1 + q] = ti[j].y;                          // arrival index of the source
        edst[o + 1 + q] = i;
    }
}

extern "C" int dagr_graph_export(const dagr_geom_t *g, int64_t N, const int32_t *perm, const int32_t *ti,
                                 const int32_t *nbr, int32_t *inv, int32_t *rowptr, int32_t *blocksums,
                                 int64_t *edge_src, int64_t *edge_dst, int64_t cap, void *stream)
{
    (void)g;
    cudaStream_t st = (cudaStream_t)stream;
    if (N <= 0) return DAGR_OK;
    k_inv_deg<<<dagr_div_up(N, 256), 256, 0, st>>>(N, perm, nbr, inv, rowptr);
    scan_exclusive(rowptr, rowptr, N, blocksums, st);
    k_export<<<dagr_div_up(N, 256), 256, 0, st>>>(N, inv, (const int2 *)ti, nbr, rowptr, edge_src, edge_dst, cap);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}
