// labels.cu -- the interframe evaluation's per-window ground truth and the packing of detections into the layout of
// dagr_evaluate_bbox (evaluate.cu), sm_90a.  Stream-ordered, no host sync; see dagr_interframe_targets and
// dagr_eval_pack_detections in include/dagr_b200.h for the data layout and the semantics restated.
//
//   k_if_count      per window: the label rows of its pair
//   scan_exclusive  -> wrow[w]: the window's first (window, row) item; wrow[Q] = items in all
//   k_if_keep       one thread per (window, label row): interpolate, crop, size filter -> keep flag
//   scan_exclusive  -> out[r]: the output row of item r (a deterministic compaction); out[R] = rows kept
//   k_if_scatter    the kept rows in xyxy with category group * K + class, and gt_off
//
//   k_pk_count      per window: its detections, or none when it has no ground truth
//   scan_exclusive  -> dt_off
//   k_pk_scatter    one thread per (window, detection slot)
#include "common.cuh"

// the last i in [0, n) with off[i] <= v (off non-decreasing, off[0] <= v)
__device__ __forceinline__ int64_t lb_last_le(const int *__restrict__ off, int64_t n, int64_t v)
{
    int64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= v) lo = mid; else hi = mid;
    }
    return lo;
}

struct IfRow {
    float x1, y1, x2, y2;
    bool keep;
};

// one label row of one window.  interpolate_tracks under NumPy 1 promotion: r = (t - t0) / (t1 - t0) in double, r and
// 1 - r rounded to float, v = v0 * (1 - r) + v1 * r in float; then Crop([0, 0], [1, 1]) (corners clamped to
// [0, W-1] x [0, H-1]), filter_small_bboxes (sqrt(h*h + w*w) > min_diag, w > min_height, h > min_height, strict) and
// convert_to_evaluation_format (x2 = x + w).  Every operation is explicitly rounded, so no contraction changes a bit.
__device__ __forceinline__ IfRow if_row(const float4 b0, const float4 b1, int64_t t, int64_t t0, int64_t t1, float xmax, float ymax,
                                        float min_h, float min_d)
{
    const double r = __ddiv_rn(__ll2double_rn(t - t0), __ll2double_rn(t1 - t0));
    const float fr = __double2float_rn(r), fq = __double2float_rn(__dsub_rn(1.0, r));
    const float x = __fadd_rn(__fmul_rn(b0.x, fq), __fmul_rn(b1.x, fr));
    const float y = __fadd_rn(__fmul_rn(b0.y, fq), __fmul_rn(b1.y, fr));
    const float w = __fadd_rn(__fmul_rn(b0.z, fq), __fmul_rn(b1.z, fr));
    const float h = __fadd_rn(__fmul_rn(b0.w, fq), __fmul_rn(b1.w, fr));
    const float cx1 = fminf(fmaxf(x, 0.f), xmax), cx2 = fminf(fmaxf(__fadd_rn(x, w), 0.f), xmax);
    const float cy1 = fminf(fmaxf(y, 0.f), ymax), cy2 = fminf(fmaxf(__fadd_rn(y, h), 0.f), ymax);
    const float cw = __fsub_rn(cx2, cx1), ch = __fsub_rn(cy2, cy1);
    const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(ch, ch), __fmul_rn(cw, cw)));
    IfRow o;
    o.x1 = cx1; o.y1 = cy1; o.x2 = __fadd_rn(cx1, cw); o.y2 = __fadd_rn(cy1, ch);
    o.keep = diag > min_d && cw > min_h && ch > min_h;
    return o;
}

struct IfArgs {
    const float4 *box0, *box1;
    const int64_t *cls, *pair_off, *pair_t, *win_pair, *win_t;
    const int32_t *win_group;
    int64_t P, L, Q, R;
    int K;
    float xmax, ymax, min_h, min_d;
};

// the pair of window w (device data: clamped to [0, P), so a bad index reads a wrong pair, never outside the tables)
__device__ __forceinline__ int64_t if_pair(const IfArgs &a, int64_t w)
{
    return min(max(__ldg(a.win_pair + w), (int64_t)0), a.P - 1);
}

__global__ void k_if_count(const IfArgs a, int *__restrict__ cnt)
{
    const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= a.Q) return;
    const int64_t p = if_pair(a, w);
    cnt[w] = a.L == 0 ? 0 : (int)max(__ldg(a.pair_off + p + 1) - __ldg(a.pair_off + p), (int64_t)0);
}

// the label row and window of item r < min(R, wrow[Q])
__device__ __forceinline__ IfRow if_item(const IfArgs &a, const int *__restrict__ wrow, int64_t r, int64_t &w, int64_t &row)
{
    w = lb_last_le(wrow, a.Q, r);
    const int64_t p = if_pair(a, w);
    row = min(max(__ldg(a.pair_off + p) + (r - wrow[w]), (int64_t)0), a.L - 1);     // device data: clamped like the pair
    return if_row(__ldg(a.box0 + row), __ldg(a.box1 + row), __ldg(a.win_t + w), __ldg(a.pair_t + 2 * p), __ldg(a.pair_t + 2 * p + 1),
                  a.xmax, a.ymax, a.min_h, a.min_d);
}

__global__ void k_if_keep(const IfArgs a, const int *__restrict__ wrow, int *__restrict__ keep)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.R) return;
    int64_t w, row;
    keep[r] = r < wrow[a.Q] ? (int)if_item(a, wrow, r, w, row).keep : 0;
}

__global__ void k_if_scatter(const IfArgs a, const int *__restrict__ wrow, const int *__restrict__ out, float4 *__restrict__ gt_box,
                             int64_t *__restrict__ gt_label, int64_t *__restrict__ gt_off)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r <= a.Q) gt_off[r] = out[min((int64_t)wrow[r], a.R)];
    if (r >= a.R || r >= wrow[a.Q] || out[r + 1] == out[r]) return;
    int64_t w, row;
    const IfRow o = if_item(a, wrow, r, w, row);
    gt_box[out[r]] = make_float4(o.x1, o.y1, o.x2, o.y2);
    gt_label[out[r]] = (int64_t)__ldg(a.win_group + w) * a.K + __ldg(a.cls + row);
}

// ---- detections -> the evaluation layout --------------------------------------------------------------------------------
__global__ void k_pk_count(const int32_t *__restrict__ ndet, const int64_t *__restrict__ gt_off, int64_t Q, int A, int *__restrict__ cnt)
{
    const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= Q) return;
    cnt[w] = __ldg(gt_off + w + 1) > __ldg(gt_off + w) ? min(max(__ldg(ndet + w), 0), A) : 0;
}

__global__ void k_pk_scatter(const float *__restrict__ det, const int32_t *__restrict__ win_group, int64_t Q, int A, int K,
                             const int *__restrict__ off, float4 *__restrict__ dt_box, float *__restrict__ dt_score,
                             int64_t *__restrict__ dt_label, int64_t *__restrict__ dt_off)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= Q) dt_off[i] = off[i];
    if (i >= Q * A) return;
    const int64_t w = i / A;
    const int j = (int)(i - w * A);
    if (j >= off[w + 1] - off[w]) return;
    const float *d = det + i * 6;
    const int64_t o = off[w] + j;
    dt_box[o] = make_float4(__ldg(d), __ldg(d + 1), __ldg(d + 2), __ldg(d + 3));
    dt_score[o] = __ldg(d + 4);
    const float lab = __ldg(d + 5);
    // Tensor.long() of the label; one outside [0, K) belongs to no category (the evaluation ignores a negative one)
    dt_label[o] = lab >= 0.f && lab < (float)K ? (int64_t)__ldg(win_group + w) * K + (int64_t)lab : -1;
}

// ---- C-ABI ------------------------------------------------------------------------------------------------------------
static int64_t lb_align(int64_t v) { return (v + 255) & ~(int64_t)255; }

// [wrow | out | blocksums] (targets) or [cnt | blocksums] (packing, R = -1)
static int64_t lb_bytes(int64_t Q, int64_t R, int64_t *o_out, int64_t *o_bs)
{
    const int64_t n = R > Q ? R : Q;
    *o_out = lb_align(4 * (Q + 1));
    *o_bs = R >= 0 ? *o_out + lb_align(4 * (R + 1)) : *o_out;
    return *o_bs + lb_align(4 * (dagr_scan_blocks(n + 1) + 2));
}

static bool if_shape_ok(int64_t P, int64_t L, int64_t Q, int64_t R, int K)
{
    return P >= 0 && L >= 0 && Q >= 0 && R >= 0 && K >= 1 && Q < (1ll << 31) - 1 && R < (1ll << 31) - 1 && L < (1ll << 31) &&
           (Q == 0 || P >= 1);
}

extern "C" int dagr_interframe_targets_workspace_bytes(int64_t n_windows, int64_t n_rows, int64_t *bytes)
{
    DAGR_CHECK_ARG(bytes != nullptr, "null bytes");
    DAGR_CHECK_ARG(n_windows >= 0 && n_rows >= 0 && n_windows < (1ll << 31) - 1 && n_rows < (1ll << 31) - 1,
                   "n_windows and n_rows in [0, 2^31 - 1)");
    int64_t a, b;
    *bytes = lb_bytes(n_windows, n_rows, &a, &b);
    return DAGR_OK;
}

extern "C" int dagr_interframe_targets(const float *box0, const float *box1, const int64_t *cls, const int64_t *pair_off,
                                       const int64_t *pair_t, int64_t n_pairs, int64_t n_labels, const int64_t *win_pair,
                                       const int64_t *win_t, const int32_t *win_group, int64_t n_windows, int K, int width,
                                       int height, float min_bbox_height, float min_bbox_diag, int64_t n_rows, void *workspace,
                                       int64_t workspace_bytes, float *gt_box, int64_t *gt_label, int64_t *gt_off, void *stream)
{
    DAGR_CHECK_ARG(if_shape_ok(n_pairs, n_labels, n_windows, n_rows, K), "n_pairs, n_labels, n_windows, n_rows >= 0, K >= 1, "
                   "n_windows and n_rows < 2^31 - 1, n_labels < 2^31, and a pair for the windows to refer to");
    DAGR_CHECK_ARG(width >= 1 && height >= 1 && width <= (1 << 24) && height <= (1 << 24), "width, height in [1, 2^24]");
    DAGR_CHECK_ARG(gt_off && workspace, "null pointer");
    DAGR_CHECK_ARG(n_windows == 0 || (pair_off && pair_t && win_pair && win_t && win_group), "null pair or window arrays");
    DAGR_CHECK_ARG(n_labels == 0 || (box0 && box1 && cls), "null label rows");
    DAGR_CHECK_ARG(n_rows == 0 || (gt_box && gt_label), "null output rows");
    DAGR_CHECK_ARG(((uintptr_t)box0 & 15) == 0 && ((uintptr_t)box1 & 15) == 0 && ((uintptr_t)gt_box & 15) == 0,
                   "boxes must be 16-byte aligned");
    int64_t o_out, o_bs;
    const int64_t need = lb_bytes(n_windows, n_rows, &o_out, &o_bs);
    DAGR_CHECK_ARG(workspace_bytes >= need && ((uintptr_t)workspace & 255) == 0,
                   "workspace smaller than dagr_interframe_targets_workspace_bytes or not 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    int *wrow = (int *)ws, *out = (int *)(ws + o_out), *bs = (int *)(ws + o_bs);
    const IfArgs a{(const float4 *)box0, (const float4 *)box1, cls, pair_off, pair_t, win_pair, win_t, win_group,
                   n_pairs, n_labels, n_windows, n_rows, K, (float)(width - 1), (float)(height - 1), min_bbox_height, min_bbox_diag};
    if (n_windows > 0) k_if_count<<<dagr_div_up(n_windows, 256), 256, 0, st>>>(a, wrow);
    scan_exclusive(wrow, wrow, n_windows, bs, st);                        // wrow[Q] = (window, row) items in all
    if (n_rows > 0) k_if_keep<<<dagr_div_up(n_rows, 256), 256, 0, st>>>(a, wrow, out);
    scan_exclusive(out, out, n_rows, bs, st);                             // out[R] = kept rows
    const int64_t grid = n_rows > n_windows + 1 ? n_rows : n_windows + 1;
    k_if_scatter<<<dagr_div_up(grid, 256), 256, 0, st>>>(a, wrow, out, (float4 *)gt_box, gt_label, gt_off);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}

extern "C" int dagr_eval_pack_workspace_bytes(int64_t n_windows, int64_t *bytes)
{
    DAGR_CHECK_ARG(bytes != nullptr, "null bytes");
    DAGR_CHECK_ARG(n_windows >= 0 && n_windows < (1ll << 31) - 1, "n_windows in [0, 2^31 - 1)");
    int64_t a, b;
    *bytes = lb_bytes(n_windows, -1, &a, &b);
    return DAGR_OK;
}

extern "C" int dagr_eval_pack_detections(const float *det, const int32_t *ndet, int64_t n_windows, int A, const int32_t *win_group,
                                         const int64_t *gt_off, int K, void *workspace, int64_t workspace_bytes, float *dt_box,
                                         float *dt_score, int64_t *dt_label, int64_t *dt_off, void *stream)
{
    DAGR_CHECK_ARG(n_windows >= 0 && n_windows < (1ll << 31) - 1 && A >= 1 && K >= 1 && n_windows * A < (1ll << 31) - 1,
                   "n_windows >= 0, A >= 1, K >= 1 and n_windows * A < 2^31 - 1");
    DAGR_CHECK_ARG(dt_off && workspace, "null pointer");
    DAGR_CHECK_ARG(n_windows == 0 || (det && ndet && win_group && gt_off && dt_box && dt_score && dt_label), "null window arrays");
    DAGR_CHECK_ARG(((uintptr_t)dt_box & 15) == 0, "dt_box must be 16-byte aligned");
    int64_t o_out, o_bs;
    const int64_t need = lb_bytes(n_windows, -1, &o_out, &o_bs);
    DAGR_CHECK_ARG(workspace_bytes >= need && ((uintptr_t)workspace & 255) == 0,
                   "workspace smaller than dagr_eval_pack_workspace_bytes or not 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    int *cnt = (int *)workspace, *bs = (int *)((char *)workspace + o_bs);
    if (n_windows > 0) k_pk_count<<<dagr_div_up(n_windows, 256), 256, 0, st>>>(ndet, gt_off, n_windows, A, cnt);
    scan_exclusive(cnt, cnt, n_windows, bs, st);                          // cnt[Q] = detections kept
    const int64_t grid = n_windows * A > n_windows + 1 ? n_windows * A : n_windows + 1;
    k_pk_scatter<<<dagr_div_up(grid, 256), 256, 0, st>>>(det, win_group, n_windows, A, K, cnt, (float4 *)dt_box, dt_score, dt_label,
                                                         dt_off);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}
