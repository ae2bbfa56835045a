/*
 * dagr_b200.h -- C-ABI of libdagr_b200.so (hand-written sm_90a CUDA kernels for DAGR's hot path).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - the library never allocates, never synchronises and never throws: callers own all
 *     buffers (workspace sizes are documented per call), every call only enqueues kernels
 *     on `stream` (a cudaStream_t passed as void*) and returns 0 or a negative code
 *     (DAGR_E_*); dagr_last_error() returns the message of the last failure on this thread;
 *   - node order: after dagr_graph_sort the event level lives in "cell-major sorted order"
 *     (position p); `perm[p]` is the arrival index the reference uses as node id.
 *
 * Each entry point cites the reference interface it replaces (paths under uzh-rpg/dagr).
 */
#ifndef DAGR_B200_H
#define DAGR_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DAGR_ABI_VERSION 3

#define DAGR_OK            0
#define DAGR_E_ARG        -1   /* bad argument / unsupported shape        */
#define DAGR_E_CUDA       -2   /* CUDA launch or runtime error            */
#define DAGR_E_UNSUPPORTED -3

#define DAGR_ELL 16            /* neighbour slots per node (K-1 = 15 used, slot 15 = degree) */
#define DAGR_KU  15            /* spline kernel slots reachable at the event level (3 x 5)   */
#define DAGR_TABW 16           /* row stride (floats) of the offset->slot-weight table       */
#define DAGR_RING_CTL 8        /* ints per stream in a streaming control block (ctl)          */

/* Staging capacities of the per-voxel event-level kernels.  Each kernel picks its instance per pool1 voxel, on the device,
 * from `total` = the number of nodes in the voxel's 3x3 neighbourhood:
 *   dagr_l1_build[_tc]     defer = 0: staged when total <= BUILD_LEAN, else the global-memory probe;
 *                          defer = 1: staged when total <= BUILD, else the dense kernel, staged when total <= BUILD_DENSE,
 *                          else the global-memory probe inside it;
 *   dagr_l1_conv_b_pool_voxel_tc / dagr_l1_conv_a_image_tc / _inc
 *                          staged when total <= CONV; above that the dense kernel when defer = 1 (staged when
 *                          total <= CONV_DENSE, else rows gathered from global memory), rows gathered in the regular kernel
 *                          when defer = 0.
 * The image conv splits a voxel with at most SPARSE_NODES own nodes over three warps (one x-slot each), in every instance.
 * wl_hdr[0] counts the voxels above BUILD_LEAN / BUILD (build, by defer) or above CONV (convs).  The build kernel's defer = 1
 * falls back to the defer = 0 launch where the dense instance does not fit the device's shared memory (dagr_l1_build). */
#define DAGR_L1_BUILD_LEAN        1536
#define DAGR_L1_BUILD             2048
#define DAGR_L1_BUILD_DENSE      12288
#define DAGR_L1_CONV              1344
#define DAGR_L1_CONV_DENSE        6144
#define DAGR_L1_SPARSE_NODES        32

/* Staging capacity (floats) of dagr_voxel_sample_max[_inc|_planes][_bf16]: a voxel stages the window of the map its events
 * can touch -- pz planes x ph rows x pw columns x C channels, derived from the voxel's corner pixels -- in shared memory when
 * pz * ph * pw * C <= DAGR_VS_SMEM_FLOATS, and reads its taps from global memory otherwise.  Staged voxels take the fast path
 * (8 channels per lane) for C in {8, 16, 32, 64, 128} and the general path (one channel per lane, 128-channel blocks)
 * otherwise.  40 KB: e.g. 2 planes x 6 x 6 x 128 channels. */
#define DAGR_VS_SMEM_FLOATS      10240

int         dagr_abi_version(void);
const char *dagr_last_error(void);

/* Geometry of one (width,height,batch,radius) configuration; tables are built on the host with
 * the same fp32 torch ops the reference uses (dagr_b200/geometry.py) and uploaded once. */
typedef struct {
    int32_t W, H, B, T;            /* sensor size, samples per batch, time window (us)               */
    int32_t r, ncell;              /* r = int(radius*W+1), ncell = (2r+1)^2   (ev_tgn.py:29)          */
    int32_t dt_us, K, Q;           /* int(radius*T), max_neighbors, max_queue_size (ev_tgn.py:22-28) */
    int32_t nx1, ny1;              /* pool1 voxel grid (pooling.py:56)                               */
    int32_t CW, CH, CP;            /* padded cell extent in pixels, CP = CW*CH                       */
    int32_t NK;                    /* number of sort keys = B*ny1*nx1*CP                             */
    const int32_t *xkey;           /* [W]  cx*CP + (x - x0[cx])                                      */
    const int32_t *ykey;           /* [H]  cy*nx1*CP + (y - y0[cy])*CW                               */
    const int8_t  *spiral;         /* [ncell][2] spiral probe order (spiral.h:1-16)                  */
    const float   *posx0;          /* [W]  fl(x / W)  (buffers.py:43)                                */
    const float   *posy0;          /* [H]  fl(y / H)                                                 */
    const int32_t *vx0;            /* [nx1+1] first pixel column of each pool1 voxel (vx0[nx1] = W)  */
    const int32_t *vy0;            /* [ny1+1] first pixel row of each pool1 voxel    (vy0[ny1] = H)  */
    const float   *tabx;           /* [2r+1][4] x factor of the slot weights: tab[c][k+3j] = tabx[dx+r][k]*taby[dy+r][j] */
    const float   *taby;           /* [2r+1][8] y factor (5 used)                                     */
} dagr_geom_t;

/* ---------------------------------------------------------------------------------------------
 * Argument contract and workspace sizes (the library never allocates; SURVEY 8(b): "workspace sizes via
 * *_workspace_bytes").  All host-only: no CUDA call is made.
 *
 *   dagr_check_config           : every shape restriction of the kernels in one place.  cin0 / cout0 = channels of
 *                                 conv_block1.conv_block1 (3 -> 16 events only, 19 -> 16 with image fusion), activation = the
 *                                 yaml `activation` key.  Returns DAGR_OK or DAGR_E_UNSUPPORTED with dagr_last_error() set.
 *   dagr_event_workspace_bytes  : byte sizes of every event-level buffer for N events (ELL leading dimension = N).
 *   dagr_pool_workspace_bytes   : byte sizes of the zero-on-entry accumulators dagr_grid_pool needs for `channels` pooled
 *                                 channels on the parent grid.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    int64_t key, tmp, count, blocksums, start, perm, ti, xyb, feat_s;   /* dagr_graph_sort[_ring]                    */
    int64_t nbr, off, cellmask, xa;                                     /* dagr_l1_build (ELL adjacency, activations)  */
    int64_t wl_hdr, wl_ids;                                             /* one dense-voxel work list (hdr zeroed)      */
    int64_t x1;                                                         /* optional per-event conv_block1 output       */
} dagr_event_ws_t;
typedef struct { int64_t acc, possum, ptmax, pcnt, pmask; } dagr_pool_ws_t;
int dagr_check_config(const dagr_geom_t *g, int64_t N, int cin0, int cout0, const char *activation);
int dagr_event_workspace_bytes(const dagr_geom_t *g, int64_t N, dagr_event_ws_t *out);
int dagr_pool_workspace_bytes(int64_t parent_cells, int channels, dagr_pool_ws_t *out);

/* ---------------------------------------------------------------------------------------------
 * a1'  denormalize_pos  (src/dagr/model/layers/ev_tgn.py:11-16):  (pos*[W,H,T] + 1e-3).int()
 * ------------------------------------------------------------------------------------------- */
int dagr_denormalize_pos(const float *pos /*[N,3]*/, int64_t N, int W, int H, int T,
                         int32_t *pos_i32 /*[N,3]*/, void *stream);
/* the input conversion of one forward in a single launch: denormalize_pos + `events.batch.int()` (ev_tgn.py:57) + the
 * polarity column x[:, 0] (row stride ldx) as a dense vector */
int dagr_prepare_events(const float *pos /*[N,3]*/, const int64_t *batch /*[N]*/, const float *x /*[N,ldx]*/, int ldx, int64_t N,
                        int W, int H, int T, int32_t *pos_i32 /*[N,3]*/, int32_t *batch_i32 /*[N]*/, float *feat /*[N]*/,
                        void *stream);

/* ---------------------------------------------------------------------------------------------
 * a2-a4  radius graph.  Replaces ev_graph_cuda.insert_in_queue_cuda + fill_edges_cuda
 * (src/dagr/graph/ev_graph.cu:82-128,241-276) and their driver (graph/utils.py:6-23,
 * ev_graph.py:63-103) for the reset=True forward.  Instead of a [B,Q,H,W] FIFO the events are
 * counting-sorted by a cell-major pixel key; a pixel's FIFO column is the tail (newest Q) of its
 * bin read backwards.
 *
 *   dagr_graph_sort   : batch i32[N], pos i32[N,3], feat f32[N] (polarity)  ->
 *                       start i32[NK+1], perm i32[N], ti i32[N,2]=(t,arrival idx),
 *                       xyb u32[N] = x | y<<12 | b<<24, feat_s f32[N]
 *                       work: key i32[N], tmp i32[N], count i32[NK+1] (MUST be zero on entry; is
 *                       zero again on exit), blocksums i32[dagr_scan_blocks(NK+1)+1]
 *                       The sort keys are int32: every sort form (and dagr_check_config) refuses a geometry whose
 *                       B*ny1*nx1*CP is >= 2^31 or differs from NK, before anything is launched.
 *   dagr_l1_build     : (below) -> nbr i32[16,N] COLUMN-MAJOR ELL: slot q of node p at [q*N+p]; slots 0..14 =
 *                       src positions in probe order, slot 15 = degree without the self loop;
 *                       off u16[16,N] (spiral cell index of each neighbour, same layout), cellmask u32[B*ny1*nx1] (bit (dcy+1)*3+(dcx+1) set when some
 *                       fine edge enters the cell from that neighbouring cell)
 *   dagr_graph_export : -> edge_index i64[2,E] exactly as the reference returns it
 *                       (dst ascending in arrival order, self loop first, then probe order);
 *                       rowptr i32[N+1] is written too; E is left in rowptr[N].
 *                       work: inv i32[N], blocksums as above (sized for N+1).
 * ------------------------------------------------------------------------------------------- */
int64_t dagr_scan_blocks(int64_t n);

int dagr_graph_sort(const dagr_geom_t *g, const int32_t *batch, const int32_t *pos, const float *feat,
                    int64_t N, int32_t *key, int32_t *tmp, int32_t *count, int32_t *blocksums,
                    int32_t *start, int32_t *perm, int32_t *ti, uint32_t *xyb, float *feat_s,
                    int32_t *flags /* i32[1], zero on entry, or NULL; [0] = 1 unless the time order is proven: the (clamped) samples
                                       come as ascending contiguous runs in arrival order, each time-sorted.  Interleaved
                                       samples set it too */,
                    void *stream);

/* Streaming form of dagr_graph_sort (BASELINE config 5; the sliding window the reference sketches with min_index,
 * src/dagr/graph/ev_graph.py:121-136, ev_graph.cu:62).  The live events of one stream sit time-sorted in ring buffers
 * batch/pos/feat of `capacity` (a power of two) slots; ctl i32[8] on the DEVICE = {head slot, live count, evicted by the last
 * push, appended by the last push, sticky overflow flag, kept count}.  Event i of the window is slot (head + i) & (capacity-1)
 * and i is its arrival index for this step.  The launch covers the capacity, so neither call depends on a host-side count:
 * a whole streaming step can be captured once and replayed as a CUDA graph.  Downstream kernels take N = capacity as the
 * leading dimension of the ELL / activation arrays.
 *   dagr_stream_push : stage i32[4 + 4*max_chunk] on the device = {n_new, t_cut, 0, 0, (x, y, t, polarity +-1) * n_new}:
 *                      evicts the prefix with t < t_cut (binary search, no data movement) and appends the chunk.
 * flags: as dagr_graph_sort, over the window in arrival order (one sample, so: [0] = 1 where the window is not time-sorted). */
int dagr_graph_sort_ring(const dagr_geom_t *g, const int32_t *batch, const int32_t *pos, const float *feat,
                         int64_t capacity, const int32_t *ctl, int32_t *key, int32_t *tmp, int32_t *count,
                         int32_t *blocksums, int32_t *start, int32_t *perm, int32_t *ti, uint32_t *xyb, float *feat_s,
                         int32_t *flags, void *stream);
int dagr_stream_push(int32_t *ctl, const int32_t *stage, int32_t *batch, int32_t *pos, float *feat, int64_t capacity,
                     int max_chunk, int sample, void *stream);

/* Multi-stream form: S independent event streams (cameras) become the S samples of one step.  Ring s owns slots
 * [s*capacity, (s+1)*capacity) of batch/pos/feat (S*capacity slots in all); `capacity` is the per-stream ring size.
 *   ctl   i32[S+1][8] on the DEVICE, zero-initialised.  Block s = {head slot inside ring s, live count, evicted by the last
 *         push, appended by the last push, sticky overflow flag, kept count, offset of the stream's window in the compact
 *         stream-major order, 0}; block S = {total live count, 0...}.  Zeroing block s resets stream s alone.
 *   stage i32[4*S + 4*S*max_chunk] on the device: header [S][4] = {n_new, t_cut, event offset, plane}, then the (x, y, t,
 *         polarity +-1) events of all streams back to back; stream s's n_new events start at event `offset`.  Word 3 is the
 *         frame plane of the stream (image fusion), ignored by the push: the *_planes entry points below read it with
 *         plane = stage + 3, plane_stride = 4.
 *   dagr_stream_push_multi : per stream, evicts the prefix with t < t_cut and appends its chunk (batch = s); then writes the
 *         window offsets (exclusive scan of the live counts) and the total.  Two launches, grids independent of the counts.
 *   dagr_graph_sort_rings  : dagr_graph_sort over the S live windows read in the compact order c < total: stream s's i-th
 *         live event has arrival index c = offset_s + i.  Outputs as dagr_graph_sort with B = S; downstream kernels take
 *         N = S*capacity.  dagr_graph_sort_ring is this sort with S = 1 and a single i32[8] block.  flags as dagr_graph_sort:
 *         the compact order is stream-major with stream s = sample s, so [0] = 1 exactly where some window is not
 *         time-sorted (a stream's first live event is not compared with the previous stream's last).
 * Limits (DAGR_E_ARG before anything is launched): no null pointer (flags may be NULL), 1 <= S <= 127, capacity a power of
 * two, S*capacity < 2^24 (sorted positions are packed in 24 bits), 1 <= max_chunk <= capacity, and for the sort S == g->B. */
int dagr_stream_push_multi(int32_t *ctl, const int32_t *stage, int32_t *batch, int32_t *pos, float *feat, int64_t capacity,
                           int streams, int max_chunk, void *stream);
int dagr_graph_sort_rings(const dagr_geom_t *g, const int32_t *batch, const int32_t *pos, const float *feat,
                          int64_t capacity, int streams, const int32_t *ctl, int32_t *key, int32_t *tmp, int32_t *count,
                          int32_t *blocksums, int32_t *start, int32_t *perm, int32_t *ti, uint32_t *xyb, float *feat_s,
                          int32_t *flags, void *stream);

/* Fused event-level build: one CTA per pool1 voxel stages the (t, arrival idx, polarity) records of the voxel's 3x3
 * neighbourhood in shared memory (three coalesced runs, thanks to the cell-major order), probes the spiral entirely on chip,
 * writes the ELL adjacency + cellmask described above and applies conv_block1.conv_block1 (SplineConv 3->16 + BN + act) to
 * the neighbours as they are found -> xa (half-major [2][N][8]), in fp32 FMA.  cellmask needs no zeroing.  With
 * p_host == NULL only the adjacency / cellmask are produced: the graph builder for callers that bring their own convs.  The
 * per-edge slot weights come from the per-axis factor tables g->tabx / g->taby.  The engine runs the tensor-core form,
 * dagr_l1_build_tc (below). */
struct dagr_l1a_params_s;
int dagr_l1_build(const dagr_geom_t *g, int64_t N, const int32_t *start, const int32_t *ti,
                  const uint32_t *xyb, const float *feat_s,
                  const struct dagr_l1a_params_s *p_host,
                  const int32_t *flags /* from the sort (any form), or NULL.  The time-bucket pruning runs only where flags[0] == 0
                                          proves the time order; NULL means the order is unknown (exact, slower) */,
                  int min_idx /* incremental mode: only events with arrival idx >= min_idx are processed and cellmask is
                                 OR-ed into its previous content; 0 = everything */,
                  int32_t *nbr, uint16_t *off, uint32_t *cellmask, float *xa,
                  int32_t *wl_hdr /* i32[2] ZERO on entry, or NULL: [0] counts the voxels whose 3x3 neighbourhood exceeds the
                                     per-voxel kernel's staging capacity (defer = 1: 2048 records; defer = 0: the lean launch with
                                     1536 records and five CTAs per SM), [1] is the dense kernel's cursor */,
                  int32_t *wl_ids /* i32[cells] or NULL: ids of those voxels when `defer` */,
                  int defer /* 1: such voxels are queued and processed by a second, persistent launch with a 12288-record staging
                               buffer; 0: they are only counted and probe global memory (slow, exact) -- a caller can watch
                               wl_hdr[0] and switch `defer` on for streams that have dense voxels.  Where the dense launch's
                               shared memory (12288 records plus the geometry's tile tables) exceeds the device's opt-in limit
                               -- large pool1 voxels at r >= 13, e.g. 1280 x 960 at radius 0.01 on an H100 -- defer = 1 runs
                               the defer = 0 launch: the same bits, wl_hdr[0] counting the voxels over 1536 records */,
                  void *stream);

/* streaming (a13): node rows live in arrival order between steps; gather (scatter=0: rows of nodes < n_old into the
 * new sorted order) / scatter (scatter=1: rows of nodes >= n_old back).  xa_sorted [2][N][8], xa_arrival [cap][16]. */
int dagr_xa_permute(int64_t N, const int32_t *perm, int n_old, float *xa_sorted, float *xa_arrival, int scatter, void *stream);

/* ---- image fusion at the event level (use_image, net.py:117-131): conv_block1 = Layer(1+16+2 -> 16) ----
 * x0 f32[3][N][8] chunk-major = [polarity, 16 bilinear samples of image_feat[0] at the event, x/W, y/H, pad];
 * sampling follows net.py:193-221 (grid_sample, align_corners=True, batch as depth).  feat_s is not read and may be NULL; any
 * other null pointer, N outside [0, 2^31) or h, w < 1 returns DAGR_E_ARG with a message before anything is launched (as for
 * every image-sampling entry point below). */
int dagr_l1_x0_image(const dagr_geom_t *g, int64_t N, const uint32_t *xyb, const float *feat_s,
                     const float *img0 /*[B,16,h,w]*/, int h, int w, float *x0, void *stream);
/* Same kernel and results, bounded by the live total start[g->NK] that the sort wrote (device data): sorted positions at or
 * beyond it are not read.  This is the form for the ring sorts, where N is the ring capacity and the positions behind the
 * live window hold stale or never-written xyb words.  feat_s is not read and may be NULL; any other null pointer, or N outside
 * [0, 2^31), returns DAGR_E_ARG with a message before anything is launched. */
int dagr_l1_x0_image_live(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s,
                          const float *img0 /*[B,16,h,w]*/, int h, int w, float *x0, void *stream);

typedef struct {
    float w[DAGR_KU][24][16];     /* slot-major spline weights, input channels padded 19 -> 24 */
    float root[24][16];
    float skip[24][16];           /* ConvBlockWithSkip.lin of conv_block2 (applied to the layer input x0) */
    float scale[16], shift[16];   /* conv_block1.norm  */
    float sscale[16], sshift[16]; /* conv_block2.norm_skip */
    int32_t relu;
} dagr_l1img_params_t;

/* per-voxel channel max (pool_mean = 0, every shipped config) or mean (pool_mean = 1, args.pooling_aggr) of image features
 * sampled at the voxel's events (sampling_skip before pool1, net.py:128-131): xg[cell*ldx + c0 + c], c < C, empty voxels -> 0.
 * Returns DAGR_E_ARG with a message before launching anything on a null pointer, N outside [0, 2^31), h or w < 1, C < 1,
 * c0 < 0 or c0 + C > ldx. */
int dagr_voxel_sample_max(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                          const float *img /*[B,C,h,w]*/, int C, int h, int w, float *xg, int ldx, int c0, int pool_mean,
                          void *stream);

int dagr_graph_export(const dagr_geom_t *g, int64_t N, const int32_t *perm, const int32_t *ti,
                      const int32_t *nbr, int32_t *inv, int32_t *rowptr, int32_t *blocksums,
                      int64_t *edge_src /*[cap]*/, int64_t *edge_dst /*[cap]*/, int64_t cap,
                      void *stream);

/* ---------------------------------------------------------------------------------------------
 * a5-a7  event-level Layer (conv_block1): Cartesian attrs + MySplineConv (LUT form) + BN + act
 * (src/dagr/model/layers/spline_conv.py:39-78, conv.py:10-72, components.py:9-35, net.py:122-126).
 * For spiral cell c, slot u of the DAGR_KU reachable spline kernel slots has the weight
 * tab[c][u] = tabx[dx+r][u%3] * taby[dy+r][u/3] (MySplineConv.init_lut's basis, spline_conv.py:27-35; geometry.py).
 * Weights are passed by value (constant bank): slot-major  w[u][cin][cout].
 * ------------------------------------------------------------------------------------------- */
typedef struct dagr_l1a_params_s {
    float w[DAGR_KU][3][16];      /* weight[slot_id[u]]  (Cin = polarity, x/W, y/H)  */
    float root[3][16];            /* lin.weight^T                                    */
    float scale[16], shift[16];   /* eval BN folded: g/sqrt(v+eps), b - m*scale      */
    int32_t relu;                 /* args.activation == relu                         */
} dagr_l1a_params_t;

typedef struct {
    float w[DAGR_KU][16][16];
    float root[16][16];
    float skip[3][16];            /* ConvBlockWithSkip.lin.mlp.weight^T             */
    float scale[16], shift[16];   /* norm                                            */
    float sscale[16], sshift[16]; /* norm_skip                                       */
    int32_t relu;
    int32_t pool_mean;            /* pool1 aggregation: 0 = max (every shipped config), 1 = mean (args.pooling_aggr) */
    /* slot u = 3*j + i is spline kernel xs[i] + 5*ys[j].  xs/ys/den describe the slot grid to tools; the kernels take
     * the basis weights from the host-built tables (geometry.py), never from in-kernel divisions (slower, measured) */
    int32_t xs[3], ys[5];
    float den_x, den_y;           /* fl32(2*M*W), fl32(2*M*H)  (spline_conv.py:28-29) */
} dagr_l1b_params_t;

/* Tensor-core form of dagr_l1_build (the engine's path).  Same arguments plus `wfrag`
 * f32[DAGR_L1A_TC_WFRAG_FLOATS] on the DEVICE: p_host->w and p_host->root as one [48][16] matrix (k = 3 u + cin for the slot
 * weights, 45 + cin for the root) in mma fragment order, split for 3xTF32, as written by dagr_l1a_tc_weights.  conv_a's
 * per-node product (45 slot inputs + 3 root inputs -> 16 channels) then runs as mma.sync TF32 (hi*hi + hi*lo + lo*hi, ~1e-6
 * relative to the fp32 sums) instead of 768 fp32 FMA per event; nbr / off / cellmask are the bits of dagr_l1_build, and every
 * node's xa row gets the same bits in every instance (lean / regular / dense, staged / global probe, any min_idx).  p_host and
 * wfrag must not be NULL (the adjacency-only form is dagr_l1_build with p_host = NULL).  Re-run dagr_l1a_tc_weights whenever the
 * weights change. */
#define DAGR_L1A_TC_WFRAG_FLOATS 1536  /* 6 k-steps x 32 lanes x 2 n-tiles x 4 */
int dagr_l1a_tc_weights(const dagr_l1a_params_t *p_host, float *wfrag_host /* f32[DAGR_L1A_TC_WFRAG_FLOATS] */);
int dagr_l1_build_tc(const dagr_geom_t *g, int64_t N, const int32_t *start, const int32_t *ti,
                     const uint32_t *xyb, const float *feat_s, const dagr_l1a_params_t *p_host, const float *wfrag,
                     const int32_t *flags, int min_idx, int32_t *nbr, uint16_t *off, uint32_t *cellmask, float *xa,
                     int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream);

/* conv_b (conv_block2: SplineConv 16->16 + BN, skip branch, act) fused with pool1 (a9, pooling.py:66-86): one CTA per pool1
 * voxel; the xa rows of the voxel's 3x3 neighbourhood (three contiguous runs in cell-major order) are staged in shared memory
 * with TMA bulk copies (cp.async.bulk + mbarrier) and pool1 is finished in the same CTA:
 * -> cnt i32[cells], pxy i32[cells,2], tmean/tmax f32[cells], xg f32[cells*ldx] (16 channels at column 0); x1 (optional, may
 * be NULL) receives the per-node activations [N,16] in sorted order.  The per-edge slot weights come from the per-axis factor
 * tables g->tabx / g->taby.  skip_pre f32[N,16] (optional): the layer's skip branch if it was produced elsewhere (image
 * fusion), else it is computed from (polarity, x/W, y/H).  min_idx > 0: incremental step, only nodes with arrival index
 * >= min_idx are convolved and `persist` f32[cells,16] carries the running per-voxel max between steps.
 * `wfrag` f32[DAGR_L1_TC_WFRAG_FLOATS] on the DEVICE: the weights of input channels 0..15 (w and root) in mma fragment order,
 * split for 3xTF32, as written by dagr_l1_tc_weights.  The slot-weight products of phase 2 and the root term run as mma.sync
 * TF32 (hi*hi + hi*lo + lo*hi, ~1e-6 relative to the fp32 sums); every node gets the same bits in every instance (regular /
 * dense, staged / gathered), and so do the per-voxel max (xg, persist), cnt, pxy, tmean and tmax.  The per-voxel MEAN
 * (pool_mean = 1) is an fp32 sum over the CTA's warps, 5 in the regular and 12 in the dense instance: a voxel over the
 * regular capacity may get other last bits with defer = 0 than with defer = 1.  Re-run dagr_l1_tc_weights whenever the
 * weights change.
 * Returns DAGR_E_ARG with a message before launching anything on a null pointer (skip_pre / persist / x1 / wl_hdr / wl_ids
 * may be NULL), N outside [0, 2^31), min_idx < 0, ldx < 16, persist with pool_mean, or min_idx > 0 without persist (the new
 * nodes alone would be pooled). */
#define DAGR_L1_TC_WFRAG_FLOATS 8192   /* 2 channel halves x 16 k-steps (15 slots + root) x 32 lanes x 2 n-tiles x 4 */
int dagr_l1_tc_weights(const float *w_host /* [DAGR_KU][cin][16] slot-major, as in the params structs */,
                       const float *root_host /* [cin][16] */, int cin /* 16 (dagr_l1b_params_t) or 24 (dagr_l1img_params_t) */,
                       float *wfrag_host /* f32[DAGR_L1_TC_WFRAG_FLOATS] */);
int dagr_l1_conv_b_pool_voxel_tc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                                 const int32_t *ti, const float *feat_s, const float *xa, const int32_t *nbr,
                                 const uint16_t *off, const dagr_l1b_params_t *p_host, const float *wfrag,
                                 const float *skip_pre /* f32[N,16] or NULL: precomputed skip branch (image path) */,
                                 int min_idx /* incremental mode: only nodes with arrival idx >= min_idx are convolved */,
                                 float *persist /* f32[cells,16] or NULL: running per-voxel max across streaming steps */,
                                 float *x1, int32_t *cnt, int32_t *pxy, float *tmean, float *tmax, float *xg,
                                 int ldx /* row stride of xg (>= 16) */,
                                 int32_t *wl_hdr /* i32[2] ZERO on entry, or NULL: [0] counts the voxels whose 3x3 neighbourhood holds
                                                    more than 1344 rows, [1] is the dense kernel's cursor */,
                                 int32_t *wl_ids /* i32[cells] or NULL */,
                                 int defer /* 1: those voxels are queued and processed by a second, persistent launch that stages up
                                              to 6144 rows (196 KB of shared memory per SM); 0: counted only, rows gathered from L2 */,
                                 void *stream);

/* conv_block1.conv_block1 on 19 input channels, image fusion.  The (polarity, x, y) channels need no gather: dagr_l1_build_tc
 * runs first with their weights (rows 0, 17, 18 of the conv, scale 1 / shift 0 / relu 0) and leaves their sums in xa; this call
 * adds the 16 sampled image channels (x0 chunk-major [2][N][8] from dagr_l1_x0_image; rows 0..15 of p_host->w / root / skip),
 * applies BN + act -> xa (half-major [2][N][8]) and writes the layer's skip branch skipv f32[N,16] = BN(Linear(x0)) (rows 16..18
 * of p_host->skip = polarity, x, y) consumed by dagr_l1_conv_b_pool_voxel_tc(skip_pre).  Same one-CTA-per-voxel, TMA-staged
 * kernel and tensor-core phase 2 as conv_b; `wfrag` as written by dagr_l1_tc_weights with cin = 24; p_host is passed by value
 * to the kernel (26 KB); wl_hdr / wl_ids / defer: the dense-voxel work list, see dagr_l1_conv_b_pool_voxel_tc.  Every node's xa
 * and skipv rows are the same bits in every instance, sparse voxels (DAGR_L1_SPARSE_NODES) included.  Returns DAGR_E_ARG with a
 * message before launching anything on a null pointer (wl_hdr / wl_ids may be NULL) or N outside [0, 2^31). */
int dagr_l1_conv_a_image_tc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s,
                            const float *x0, const int32_t *nbr, const uint16_t *off, const dagr_l1img_params_t *p_host,
                            const float *wfrag, float *xa, float *skipv, int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream);

/* ---- incremental stream steps with image fusion (a13 with use_image) ----
 * dagr_l1_conv_a_image_inc: dagr_l1_conv_a_image_tc for an append-only stream step.  Only nodes whose arrival index
 * ti[p].y (int32[N][2] from the sort) is >= min_idx are convolved: their xa rows (the probe's event-channel sums, as
 * dagr_l1_build with the same min_idx left them) are finished and their skipv rows written.  The xa rows of older nodes hold
 * the final activations gathered from arrival storage (dagr_xa_permute) and are left untouched, skipv rows of older nodes
 * are not written.  x0 must hold the samples of EVERY node (a new node's conv reads its older neighbours' x0).  min_idx = 0
 * gives the bits of dagr_l1_conv_a_image_tc.
 * dagr_voxel_sample_max_inc: dagr_voxel_sample_max (max only) with a running per-voxel max persist f32[cells][C] across
 * steps.  min_idx = 0 samples every event, seeds persist (-inf for empty voxels) and gives the bits of dagr_voxel_sample_max;
 * min_idx > 0 samples only the events with arrival index >= min_idx and combines their max with persist; a voxel without
 * such events copies persist to xg and stages nothing.
 * Both return DAGR_E_ARG with a message before launching anything on a null pointer (wl_hdr / wl_ids may be NULL), a
 * negative min_idx, N outside [0, 2^31), c0 + C > ldx or pool_mean != 0 (the stream's running aggregate is a max). */
int dagr_l1_conv_a_image_inc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                             const float *feat_s, const float *x0, const int32_t *nbr, const uint16_t *off,
                             const dagr_l1img_params_t *p_host, const float *wfrag, int min_idx, float *xa, float *skipv,
                             int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream);
int dagr_voxel_sample_max_inc(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                              const float *img /*[B,C,h,w]*/, int C, int h, int w, int min_idx, float *persist, float *xg, int ldx,
                              int c0, int pool_mean, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Coarse levels live on dense voxel grids [B, ny, nx]: per cell  valid, pixel position, features,
 * and an 8-neighbour in-edge mask (bit (dcy+1)*3+(dcx+1), src cell = dst cell + (dcx,dcy)).
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t nx, ny, B;             /* grid                                            */
    int32_t W, H;                  /* sensor size                                     */
    const float *posxr;            /* [W] fl(k * fl(1/W))  (pooling.py:47-49)         */
    const float *posyr;            /* [H]                                             */
} dagr_grid_t;

/* cat(x, pos[:, :2]) (net.py:135-136 etc.): xin[cells, Cx+2] */
int dagr_grid_cat_pos(const dagr_grid_t *gr, const int32_t *cnt, const int32_t *pxy, const float *x,
                      int Cx, float *xin, void *stream);

/* a6 on a voxel grid: MySplineConv (basis form evaluated at the exact integer pixel offsets, which is
 * what message_lut computes, spline_conv.py:39-47) + root + bias, then optional eval-BN, optional
 * residual `skip` (already BN'd, [cells,Cout]) and optional relu -- i.e. ConvBlock / ConvBlockWithSkip
 * (conv.py:10-56).
 *   weight f32[25,Cin,Cout], rootT f32[Cin,Cout] (= lin.weight^T), bias f32[Cout]|NULL,
 *   scale/shift f32[Cout]|NULL (folded eval BN)
 *   attr = d/den + 0.5 with den_x = fl(2*M*W), den_y = fl(2*M*H)  (spline_conv.py:28-29)
 */
int dagr_grid_conv(const dagr_grid_t *gr, const int32_t *cnt, const int32_t *pxy, const uint32_t *mask,
                   const float *xin, int ldin /* row stride of xin in floats (0 = Cin): the input may be a column block of a
                                                 wider array, e.g. one half of the fused cls_conv|reg_conv output */,
                   int Cin, int Cout, const float *weight, const float *rootT,
                   const float *bias, const float *scale, const float *shift, const float *skip,
                   int relu, float den_x, float den_y, float *out, void *stream);
/* which kernel the last successful dagr_grid_conv call on this thread launched: 16 for the large-grid tiled kernel, the
 * voxels per CTA of the split-K kernel (4 or 1), 0 for the one-warp-per-voxel kernel, -1 before any such call (tests
 * assert the instance a shape reaches) */
int dagr_grid_conv_last_instance(void);

/* y = BN(x @ W^T) on valid cells (Linear + BatchNormData of ConvBlockWithSkip, conv.py:41-52);
 * wT f32[Cin,Cout] */
int dagr_grid_linear_bn(int64_t cells, const int32_t *cnt, const float *xin, int Cin, int Cout,
                        const float *wT, const float *scale, const float *shift,
                        float *out, void *stream);

/* a9 on grids (pool2..4): scatter children into parent voxels. aggr: 0 = max, 1 = mean.
 * cellx/celly: [W]/[H] pixel -> parent voxel index LUT (fp32-exact, geometry.py).
 * accumulators (all MUST be zero on entry): accmax u32[cellsP*C] (aggr 0) | accsum f64[cellsP*C]
 * (aggr 1), possum f64[cellsP,3], ptmax u32[cellsP], pcnt i32[cellsP], pmask u32[cellsP];
 * err_flag i32[1] is set to 1 if a coarse edge would span more than one voxel. */
int dagr_grid_pool(const dagr_grid_t *child, const dagr_grid_t *parent, const int32_t *cellx,
                   const int32_t *celly, const int32_t *cnt, const int32_t *pxy, const float *tmean,
                   const float *tmax, const uint32_t *mask, const float *x, int C, int aggr,
                   uint32_t *accmax, double *accsum, double *possum, uint32_t *ptmax, int32_t *pcnt,
                   uint32_t *pmask, int32_t *err_flag, void *stream);

int dagr_grid_pool_finalize(const dagr_grid_t *parent, int C, int aggr, const uint32_t *accmax,
                            const double *accsum, const double *possum, const uint32_t *ptmax,
                            const int32_t *pcnt, int32_t *pxy, float *tmean, float *tmax, float *x,
                            void *stream);

/* keep_temporal_ordering (pooling.py:69-72): drop in-edges with t_max[dst] <= t_max[src] */
int dagr_grid_temporal_filter(const dagr_grid_t *gr, const int32_t *cnt, const float *tmax,
                              uint32_t *mask, void *stream);

/* a10 to_dense (spline_conv.py:80-107): grid-major [cells, C] -> dense [B, C, ny, nx] (+= add, optional) */
int dagr_grid_to_dense(const dagr_grid_t *gr, const int32_t *cnt, const float *x, int C, int ldx /* row stride of x, 0 = C */,
                       const float *add /*[B,C,ny,nx] or NULL*/, float *dense, void *stream);

/* to_dense of the three prediction convs + the CNN head maps (dagr.py:219-222) + collect_outputs + decode_outputs of one
 * scale in one launch: cls f32[cells, ldc] (nc used), regobj f32[cells, ldr] = (reg[4], obj[1]) as written by ONE conv over the
 * concatenated reg_pred|obj_pred weights; add_* [B,C,ny,nx] or NULL -> out[B, A, 5+nc] rows [a0, a0 + ny*nx) */
int dagr_head_finish(const dagr_grid_t *gr, const int32_t *cnt, const float *cls, int ldc, const float *regobj, int ldr,
                     const float *add_cls, const float *add_reg, const float *add_obj, int nc, int stride, int a0, int A,
                     float *out, void *stream);

/* a11 postprocess_network_output + batched_nms_coordinate_trick (model/utils.py:25-33,61-110).
 * pred f32[B,A,5+nc] (decoded, cxcywh) -> det f32[B,A,6] = (x1,y1,x2,y2,score,label) compacted in
 * descending-score order, ndet i32[B].  One CTA per image, A <= 256.  torchvision.ops.nms semantics bit for bit: the
 * IoU, areas, xyxy corners and obj * cls^2 round every step on its own (no FMA), as torchvision's CPU kernel and the
 * reference's torch code do,
 * compared against the fp32 nms_thre / conf_thre as the reference's torch code does (torchvision compares the IoU with
 * the double threshold: the same decisions wherever fl32(nms_thre) <= nms_thre, as at 0.65); ties in score go to the
 * lower anchor, ties in class to the first class.
 * Returns DAGR_E_ARG with a message before launching anything on a null pred / det / ndet, nc < 1, A outside [1, 256]
 * or B < 0; B == 0 returns DAGR_OK without a launch. */
int dagr_postprocess_nms(const float *pred, int B, int A, int nc, float conf_thre, float nms_thre,
                         int width, int height, int filtering, float *det, int32_t *ndet, void *stream);

/* a8 sample_features (net.py:193-221): bilinear, align_corners=True, batch as depth.
 * img f32[Bi,C,h,w]; positions given as normalised floats; out[n, ldo] columns [c0, c0+C).  Every sample_features form
 * (plain, _planes, _bf16) returns DAGR_E_ARG with a message before launching anything on a null pointer, n outside [0, 2^31),
 * Bi, C, h or w < 1, c0 < 0 or c0 + C > ldo. */
int dagr_sample_features(const float *img, int Bi, int C, int h, int w, const float *posx, const float *posy,
                         const int32_t *bidx, int64_t n, int width, int height, float *out, int ldo, int c0,
                         void *stream);

/* Plane mode of the image kernels (several hybrid cameras as the samples of one streaming step, each with its own frame):
 * the image is a plane array [nplanes][C][h][w] and sample b reads plane[b * plane_stride] alone, sampled as a batch of
 * one -- the bits a B = 1 forward gives that sample with that plane as its image (the batched forward samples with the batch
 * index as a third grid_sample coordinate, which mixes neighbouring planes where it is not an integer).  Plane values are
 * device data: the kernels clamp them to [0, nplanes).  Every *_planes entry point returns DAGR_E_ARG with a message before
 * launching anything on a null pointer (feat_s may be NULL), nplanes < 1, plane_stride < 1 or N outside [0, 2^31).
 *   dagr_l1_x0_image_planes      : dagr_l1_x0_image_live (bounded by the live total start[g->NK]) with img0 [nplanes,16,h,w].
 *   dagr_voxel_sample_max_planes : dagr_voxel_sample_max with img [nplanes,C,h,w]; a voxel's window is staged from its one
 *                                  plane; also refuses c0 + C > ldx.
 *   dagr_sample_features_planes  : dagr_sample_features with img [nplanes,C,h,w]; node i samples plane[bidx[i] * stride].
 *   dagr_head_finish_planes      : dagr_head_finish with add_* [nplanes,C,ny,nx] (all three required); the maps of sample b
 *                                  are read at plane[b * stride]. */
int dagr_l1_x0_image_planes(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s,
                            const float *img0, int h, int w, int nplanes, const int32_t *plane, int plane_stride, float *x0,
                            void *stream);
int dagr_voxel_sample_max_planes(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *img, int C,
                                 int h, int w, int nplanes, const int32_t *plane, int plane_stride, float *xg, int ldx, int c0,
                                 int pool_mean, void *stream);
int dagr_sample_features_planes(const float *img, int nplanes, const int32_t *plane, int plane_stride, int C, int h, int w,
                                const float *posx, const float *posy, const int32_t *bidx, int64_t n, int width, int height,
                                float *out, int ldo, int c0, void *stream);
int dagr_head_finish_planes(const dagr_grid_t *gr, const int32_t *cnt, const float *cls, int ldc, const float *regobj, int ldr,
                            const float *add_cls, const float *add_reg, const float *add_obj, int nc, int stride, int a0, int A,
                            int nplanes, const int32_t *plane, int plane_stride, float *out, void *stream);

/* bf16 NHWC maps (the taps of the bf16 image branch, DAGR.image_precision = "bf16"): each sampling entry point above has a
 * _bf16 form that takes the map as `const void *` to bf16 in NHWC order -- [B][h][w][C], or [nplanes][h][w][C] for the
 * _planes forms; a torch tensor [B, C, h, w] in channels_last memory format -- with its (C, h, w), and otherwise the same
 * arguments.  Each returns exactly the floats its fp32 form returns on the NCHW fp32 upcast of the same map (bf16 -> fp32
 * is exact; the taps, their order and the fp32 arithmetic are those of the fp32 form).  Every _bf16 entry point returns
 * DAGR_E_ARG with a message before launching anything on a null pointer (feat_s may be NULL), N outside [0, 2^31), h or
 * w < 1, and as its _planes / _inc sibling on nplanes < 1, plane_stride < 1, min_idx < 0, c0 + C > ldx or pool_mean with
 * _inc.  The x0 forms take C and require C == 16. */
int dagr_l1_x0_image_bf16(const dagr_geom_t *g, int64_t N, const uint32_t *xyb, const float *feat_s,
                          const void *img0 /*bf16 [B,h,w,16]*/, int C, int h, int w, float *x0, void *stream);
int dagr_l1_x0_image_live_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s,
                               const void *img0 /*bf16 [B,h,w,16]*/, int C, int h, int w, float *x0, void *stream);
int dagr_l1_x0_image_planes_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const float *feat_s,
                                 const void *img0 /*bf16 [nplanes,h,w,16]*/, int C, int h, int w, int nplanes, const int32_t *plane,
                                 int plane_stride, float *x0, void *stream);
int dagr_voxel_sample_max_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                               const void *img /*bf16 [B,h,w,C]*/, int C, int h, int w, float *xg, int ldx, int c0, int pool_mean,
                               void *stream);
int dagr_voxel_sample_max_inc_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb, const int32_t *ti,
                                   const void *img /*bf16 [B,h,w,C]*/, int C, int h, int w, int min_idx, float *persist, float *xg,
                                   int ldx, int c0, int pool_mean, void *stream);
int dagr_voxel_sample_max_planes_bf16(const dagr_geom_t *g, int64_t N, const int32_t *start, const uint32_t *xyb,
                                      const void *img /*bf16 [nplanes,h,w,C]*/, int C, int h, int w, int nplanes, const int32_t *plane,
                                      int plane_stride, float *xg, int ldx, int c0, int pool_mean, void *stream);
int dagr_sample_features_bf16(const void *img /*bf16 [Bi,h,w,C]*/, int Bi, int C, int h, int w, const float *posx, const float *posy,
                              const int32_t *bidx, int64_t n, int width, int height, float *out, int ldo, int c0, void *stream);
int dagr_sample_features_planes_bf16(const void *img /*bf16 [nplanes,h,w,C]*/, int nplanes, const int32_t *plane, int plane_stride,
                                     int C, int h, int w, const float *posx, const float *posy, const int32_t *bidx, int64_t n,
                                     int width, int height, float *out, int ldo, int c0, void *stream);

/* ---------------------------------------------------------------------------------------------
 * a14  asy_tools (src/dagr/asynchronous/asy_tools/main.cu:239-244), same argument meaning.
 * masked_isdiff writes kept[i] = idx[i] or -1 (the reference clobbers `indices` in place, :30-37);
 * compaction is the caller's job exactly as in main.cu:124.
 * The outputs equal the reference kernels' bit for bit as nvcc builds them (FMA contraction on):
 * masked_lin accumulates with fmaf in channel order and adds the bias last; masked_inplace_bn ends
 * in one fmaf(d, weight, bias); masked_isdiff tests |a - b| > fmaf(rtol, b, atol) with b signed.
 * Precondition: the K indices are distinct.  With duplicates, masked_lin with add = 1 (and every
 * op writing the same row twice) races, as the reference kernels do.
 * DAGR_E_ARG before any launch: K < 0, Cin / Cout / C < 1, or a NULL pointer when K > 0 (only
 * masked_lin's bias may be NULL).
 * ------------------------------------------------------------------------------------------- */
int dagr_masked_lin(const int64_t *idx, int64_t K, const float *x_in, float *x_out, const float *weight,
                    const float *bias /*or NULL*/, int Cin, int Cout, int add, void *stream);
int dagr_masked_inplace_bn(const int64_t *idx, int64_t K, const float *x, float *x_out, const float *mean,
                           const float *var, const float *weight, const float *bias, int C, float eps,
                           void *stream);
int dagr_masked_isdiff(int64_t *idx_inout, int64_t K, const float *a, const float *b, int C, float atol,
                       float rtol, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Event ingest on the device (SURVEY 8(f) rank 1): what the reference does on the CPU between the raw DSEC stream and
 * the graph builder.
 *
 *   dagr_downsample_events : scripts/downsample_events.py:91-124 (downsample_events + the numba loop
 *       _filter_events_resize).  x,y u16[N] at the input resolution, p i8[N] in {-1,+1}, events in time order;
 *       fx = int(in_w/out_w), fy = int(in_h/out_h); change_map f32[out_h*out_w] is the per-output-pixel accumulator that
 *       the script carries from chunk to chunk (in/out).  mask u8[N] (out) = 1 where the event passes.
 *       work: cell,tmp,sorted i32[N]; count i32[out_h*out_w] (MUST be zero on entry; is zero again on exit);
 *       start i32[out_h*out_w+1]; blocksums i32[dagr_scan_blocks(max(N, out_h*out_w))+2].  Every mask byte is written.
 *       Output cell (min(x / fx, out_w - 1), min(y / fy, out_h - 1)): the reference would index out of bounds.
 *   dagr_compact_events   : events[mask] with x/fx, y/fy as (x / fx).astype(uint16) (:102-104); order preserved; any
 *       non-zero mask byte keeps its event.  work: flag i32[N], pos i32[N+1], blocksums i32[dagr_scan_blocks(N)+2];
 *       n_out i32[1] (device) = number kept.  Nothing is written to xo, yo, to, po past n_out.
 *   dagr_ingest_events    : one sample: keep t < t_cut (dsec_data.py:177-179) and y < H (:142-143), t = T + t - t[-1]
 *       (:144-145) where t[-1] is the t of the last kept event in array order (the events need not be time-sorted, and
 *       t may be negative), polarity 2p-1 when p_is_01 (:146; else p as is), int16/int32 casts (data/utils.py:12-13:
 *       x, y >= 2^15 and relative t outside int32 wrap), fp32 normalisation by [W,H,T] (utils/buffers.py:41-43) and
 *       denormalisation (ev_tgn.py:15-16) -> batch i32[M] (= sample), pos i32[M,3], polarity f32[M]: the inputs of
 *       dagr_graph_sort.  work: flag i32[N], pos i32[N+1], blocksums i32[dagr_scan_blocks(N)+2], tlast u64[1] (the
 *       index of the last kept event, -1 when none).
 * All three return DAGR_E_ARG with a message before anything is launched on a null pointer (the N-long rows may be NULL
 * when N = 0), N outside [0, 2^31), fx or fy < 1, out_w or out_h < 1, out_w * out_h >= 2^31, or W, H or T < 1.
 * ------------------------------------------------------------------------------------------- */
int dagr_downsample_events(const uint16_t *x, const uint16_t *y, const int8_t *p, int64_t N, int fx, int fy,
                           int out_w, int out_h, float *change_map, int32_t *cell, int32_t *tmp, int32_t *sorted,
                           int32_t *count, int32_t *start, int32_t *blocksums, uint8_t *mask, void *stream);
int dagr_compact_events(const uint8_t *mask, int64_t N, const uint16_t *x, const uint16_t *y, const int64_t *t,
                        const int8_t *p, int fx, int fy, int32_t *flag, int32_t *pos, int32_t *blocksums,
                        uint16_t *xo, uint16_t *yo, int64_t *to, int8_t *po, int32_t *n_out, void *stream);
int dagr_ingest_events(const uint16_t *x, const uint16_t *y, const int64_t *t, const int8_t *p, int64_t N,
                       int p_is_01, int W, int H, int T, int64_t t_cut, int sample, int32_t *flag, int32_t *pos,
                       int32_t *blocksums, unsigned long long *tlast, int32_t *batch_out, int32_t *pos_out,
                       float *feat_out, int32_t *n_out, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Windows of one recording (dagr_b200.sequence): many time windows of a time-sorted recording as the samples of batched
 * forwards.
 *
 *   dagr_window_bounds : t i64[N] sorted (non-decreasing); window q = [t_begin[q], t_end[q]) (i64[Q] each, on the device)
 *       -> begin[q] = lower_bound(t, t_begin[q]), end[q] = lower_bound(t, t_end[q]) (i32[Q]), one thread per window.  This
 *       is the live-window rule of the streaming rings: an event with t == t_end - window_us is live, one with t == t_end is
 *       not.  Returns DAGR_E_ARG with a message before anything is launched on a null pointer (t may be NULL when N = 0,
 *       the Q-long rows when Q = 0), N outside [0, 2^31) or Q outside [0, 2^31).
 *   dagr_window_gather : the G windows {begin[g], end[g]} (i32[G] on the device, G in [1, 255]; end < begin counts as
 *       empty) of the recording x, y u16[N], t i64[N], p i8[N] -> the inputs of dagr_graph_sort, window g's events in
 *       recording order at rows [offsets[g], offsets[g + 1]): batch i32 = g, pos i32[., 3] = (x, y, t - t_base) (t - t_base
 *       is kept in its low 32 bits), feat f32 = 2p - 1 when p_is_01, else p as is.  offsets i64[G + 1] (out) = the exclusive
 *       scan of the window sizes, offsets[G] their total.  Windows may overlap, repeat or be empty.  `total` = the rows the
 *       outputs hold (the block total the caller read back): no row at or past it is written.  One CTA per 1024 rows, no
 *       atomics.  Returns DAGR_E_ARG with a message before anything is launched on a null pointer (the N-long rows may be
 *       NULL when N = 0, the output rows when total = 0), N outside [0, 2^31), G outside [1, 255] or total outside [0, 2^24)
 *       (dagr_graph_sort packs sorted positions in 24 bits).
 * ------------------------------------------------------------------------------------------- */
int dagr_window_bounds(const int64_t *t, int64_t N, const int64_t *t_begin, const int64_t *t_end, int64_t Q, int32_t *begin,
                       int32_t *end, void *stream);
int dagr_window_gather(const uint16_t *x, const uint16_t *y, const int64_t *t, const int8_t *p, int64_t N, const int32_t *begin,
                       const int32_t *end, int G, int64_t t_base, int p_is_01, int64_t total, int32_t *batch_out, int32_t *pos_out,
                       float *feat_out, int64_t *offsets, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Streaming ingest: raw sensor chunks of S cameras -> the stage of dagr_stream_push / dagr_stream_push_multi, as one
 * launch of S CTAs whose grid depends on no count (capturable in the streaming step's CUDA graph; no host sync).
 *
 *   raw_stage i32[4*S + 2*S*max_raw] on the DEVICE: header [S][4] = {n_raw, t_cut, event offset, plane}, then the raw
 *         events of all streams back to back, 8 bytes each: word 0 = x | y << 16 | polarity << 31 (x < 2^16, y < 2^15,
 *         polarity bit 1 = +1, 0 = -1), word 1 = t in the stream's rebased time (int32 us).  Stream s's n_raw events start
 *         at event `offset`.  t_cut is in rebased time; t_cut and the plane word are carried to the output unchanged.
 *   change_map f32[S][out_h][out_w] (in/out): the per-output-pixel accumulators of the down-sampler, carried from step to
 *         step (scripts/downsample_events.py:146-153); zero a stream's map to restart it (the script starts every recording
 *         with change_map = None).  Untouched when fx = fy = 1.
 *   stage i32[4*S + 4*S*max_chunk] (out): header {n_kept, t_cut, s * max_chunk, plane}, then stream s's kept events at
 *         event s * max_chunk as (x / fx, y / fy, t, polarity +-1) rows: the input of the push.
 * Per stream, in arrival order: output cell (min(x / fx, out_w - 1), min(y / fy, out_h - 1)); the reference's per-cell
 * accumulator walk (the arithmetic of dagr_downsample_events, the same device function); the kept events in arrival
 * order; crop to y / fy < crop_h (dsec_data.py:142-143).  A cell with many events in one chunk is walked serially.
 * Limits (DAGR_E_ARG before anything is launched): no null pointer; 1 <= S <= 127; fx, fy >= 1; out_w * fx <= 2^16 and
 * out_h * fy <= 2^15 (the raw record); out_w * out_h <= DAGR_INGEST_MAX_CELLS unless fx = fy = 1 (32-bit sort key
 * cell << 14 | arrival index); 1 <= crop_h <= out_h; 1 <= max_raw <= DAGR_INGEST_MAX_RAW (the sort runs in shared
 * memory); max_raw <= max_chunk.  n_raw is clamped to [0, max_raw] on the device.
 * ------------------------------------------------------------------------------------------- */
#define DAGR_INGEST_MAX_RAW   16384       /* raw events per stream per step                           */
#define DAGR_INGEST_MAX_CELLS (1 << 18)   /* output cells of a down-sampling grid (fx * fy > 1)       */
int dagr_stream_ingest(const int32_t *raw_stage, int streams, int max_raw, int fx, int fy, int out_w, int out_h, int crop_h,
                       float *change_map, int32_t *stage, int max_chunk, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Camera frames: the reference's DSEC.preprocess_image (dsec_data.py:149-154) on the device, bit for bit: crop to
 * scale * out_h rows, cv2.resize(INTER_CUBIC) by the integer factor `scale`, HWC -> CHW.
 *
 *   frames u8[nframes][src_h][src_w][3] contiguous, the camera's channel order (passed through unchanged).
 *   out_u8 u8[nframes][3][out_h][out_w] (the reference's data.image), or
 *   out_f32 f32[nframes][3][out_h][out_w] = lut[byte]; lut f32[256] on the device, built by the caller as
 *         torch.arange(256, dtype=uint8).float() / 255.0 (the bits of format_data's `.float() / 255.0`).
 * Exactly one of out_u8 / out_f32 is given.  Integer arithmetic: odd scale picks source pixel scale * d + (scale - 1) / 2;
 * even scale sums taps sx - 1 .. sx + 2 (sx = scale * d + scale / 2 - 1, clamped to the cropped frame) with weights
 * [-3, 19, 19, -3] / 32 per axis and rounds the sum half to even, saturated to [0, 255].
 * Limits (DAGR_E_ARG before anything is launched): no null frames / lut (with out_f32); 1 <= nframes <= 65535;
 * out_w >= 1, 1 <= out_h <= 65535; scale >= 1; src_w == scale * out_w; src_h >= scale * out_h; src_h * src_w * 3 < 2^31.
 * ------------------------------------------------------------------------------------------- */
int dagr_frame_preprocess(const uint8_t *frames, int nframes, int src_h, int src_w, int scale, int out_h, int out_w,
                          uint8_t *out_u8, float *out_f32, const float *lut, void *stream);

/* ---------------------------------------------------------------------------------------------
 * COCO bbox evaluation: the reference's DetectionBuffer.compute / evaluate_detection (src/dagr/utils/buffers.py:118-123,
 * coco_eval.py:64-230), i.e. pycocotools' COCOeval (evaluate + accumulate) with maxDets = 100, on the device.
 *
 *   gt_box f32[n_gt][4] / dt_box f32[n_det][4]  xyxy, 16-byte aligned; gt_label / dt_label i64 (the class index, taken
 *         modulo 2^32 like the reference's uint32 class_id); dt_score f32[n_det].
 *   gt_off / dt_off i64[n_images + 1]: image i owns GT rows [gt_off[i], gt_off[i+1]) and detection rows [dt_off[i], dt_off[i+1]).
 *   params_host: the float64 thresholds and area ranges (np.linspace(.5, .95, 10), np.linspace(0, 1, 101), COCO areaRng).
 *   precision f64[10][101][K][4] and recall f64[10][K][4] (out): COCOeval.eval['precision'|'recall'][..., maxDets = 100].
 * Semantics: x, y, w = x2 - x1, h = y2 - y1 and area = w * h in float32; images without GT contribute nothing; per (image,
 * class) the detections are ranked by descending score (stable) and the first 100 kept; IoU is bbIou in double; greedy
 * matching per area range and IoU threshold as evaluateImg (GTs outside the range last, unmatched detections outside it
 * ignored); per (class, area) the kept detections of every image, stably sorted by score, give cumulative tp / fp,
 * rc = tp / npig, pr = tp / (fp + tp + 2^-52), the right-to-left max envelope and searchsorted(rc, rec_thrs, 'left').
 * A class without a GT inside the area range keeps -1.  Boxes must be finite.  One warp per (image, class) stages up to 32
 * GTs and their IoU table; more GTs of one class in one image take the same arithmetic from global memory.
 * workspace: dagr_eval_workspace_bytes bytes, 256-byte aligned, no initialisation.
 * Limits (DAGR_E_ARG before anything is launched): n_images >= 1, 1 <= K <= 65535, n_images * K < 2^31 - 1,
 * n_det < 2^31, n_images < 2^31 / 100, no null pointer (row pointers may be NULL when their count is 0).
 * ------------------------------------------------------------------------------------------- */
typedef struct {
    double iou_thrs[10];
    double rec_thrs[101];
    double area_rng[4][2];         /* all, small, medium, large: [lo, hi], a box is outside when area < lo or area > hi */
} dagr_eval_params_t;
int dagr_eval_workspace_bytes(int64_t n_images, int K, int64_t n_gt, int64_t n_det, int64_t *bytes);
int dagr_evaluate_bbox(const float *gt_box, const int64_t *gt_label, const int64_t *gt_off, const float *dt_box,
                       const float *dt_score, const int64_t *dt_label, const int64_t *dt_off, int64_t n_images, int K,
                       int64_t n_gt, int64_t n_det, const dagr_eval_params_t *params_host, void *workspace,
                       int64_t workspace_bytes, double *precision, double *recall, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Interframe evaluation (the reference's scripts/run_test_interframe.py): the ground truth of every window and the
 * detections of every window in the layout of dagr_evaluate_bbox, with one category block per group (offset), so that
 * one evaluate call over K' = n_groups * K categories equals one call per group.
 *
 * dagr_interframe_targets: window w = (pair win_pair[w], time win_t[w], group win_group[w]).
 *   box0 / box1 f32[n_labels][4] xywh (16-byte aligned): the preprocessed labels of the pair's first and second frame,
 *         paired row by row and sorted by track id; pair p owns rows [pair_off[p], pair_off[p+1]); cls i64[n_labels] the
 *         class index (from the first frame); pair_t i64[n_pairs][2] = (t0, t1), t0 < t1.
 *   Per window and row, as dsec_data.interpolate_tracks under NumPy 1 promotion: r = (t - t0) / (t1 - t0) in double, r and
 *   1 - r rounded to float, v = v0 * (1 - r) + v1 * r in float for x, y, w, h; then augment.Crop([0, 0], [1, 1]) (both
 *   corners clamped to [0, width-1] x [0, height-1]), filter_small_bboxes (float sqrt(h*h + w*w) > min_bbox_diag,
 *   w > min_bbox_height, h > min_bbox_height) and x2 = x + w, y2 = y + h.  Every operation is correctly rounded.
 *   Out: the kept rows of every window in window order, each window's rows in table order: gt_box f32[n_rows][4] xyxy
 *   (16-byte aligned), gt_label i64[n_rows] = win_group * K + cls, gt_off i64[n_windows + 1].
 *   n_rows: the capacity, the sum over the windows of their pairs' row counts (rows past it are not evaluated).
 *   win_pair and pair_off are device data the launch cannot check: a pair index is clamped to [0, n_pairs) and a row
 *   index to [0, n_labels).
 *   workspace: dagr_interframe_targets_workspace_bytes bytes, 256-byte aligned, no initialisation.
 *   Limits (DAGR_E_ARG before anything is launched): counts >= 0, K >= 1, n_windows and n_rows < 2^31 - 1,
 *   n_labels < 2^31, n_pairs >= 1 when n_windows > 0, 1 <= width, height <= 2^24, no null pointer where a count is > 0.
 *
 * dagr_eval_pack_detections: det f32[n_windows][A][6] (x1, y1, x2, y2, score, label) and ndet i32[n_windows] as
 *   Engine.postprocess / SequenceDetector return them.  A window with ground truth (gt_off[w+1] > gt_off[w]) keeps its
 *   first min(max(ndet, 0), A) detections, one without keeps none (an image without GT contributes nothing).
 *   Out: dt_box f32[n_windows * A][4] (16-byte aligned), dt_score f32[.], dt_label i64[.] = win_group * K + (long)label,
 *   or -1 (no category) for a label outside [0, K); dt_off i64[n_windows + 1].
 *   workspace: dagr_eval_pack_workspace_bytes bytes, 256-byte aligned, no initialisation.
 *   Limits (DAGR_E_ARG): n_windows >= 0, A >= 1, K >= 1, n_windows * A < 2^31 - 1, no null pointer when n_windows > 0.
 * ------------------------------------------------------------------------------------------- */
int dagr_interframe_targets_workspace_bytes(int64_t n_windows, int64_t n_rows, int64_t *bytes);
int dagr_interframe_targets(const float *box0, const float *box1, const int64_t *cls, const int64_t *pair_off,
                            const int64_t *pair_t, int64_t n_pairs, int64_t n_labels, const int64_t *win_pair,
                            const int64_t *win_t, const int32_t *win_group, int64_t n_windows, int K, int width, int height,
                            float min_bbox_height, float min_bbox_diag, int64_t n_rows, void *workspace,
                            int64_t workspace_bytes, float *gt_box, int64_t *gt_label, int64_t *gt_off, void *stream);
int dagr_eval_pack_workspace_bytes(int64_t n_windows, int64_t *bytes);
int dagr_eval_pack_detections(const float *det, const int32_t *ndet, int64_t n_windows, int A, const int32_t *win_group,
                              const int64_t *gt_off, int K, void *workspace, int64_t workspace_bytes, float *dt_box,
                              float *dt_score, int64_t *dt_label, int64_t *dt_off, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* DAGR_B200_H */
