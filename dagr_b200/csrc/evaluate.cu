// evaluate.cu -- COCO bbox evaluation (mAP) of the reference's DetectionBuffer.compute (src/dagr/utils/buffers.py:118-123,
// coco_eval.py:64-230 with pycocotools' COCOeval semantics), sm_90a.  Stream-ordered, no host sync; see dagr_evaluate_bbox
// in include/dagr_b200.h for the data layout and the semantics restated.
//
//   k_eval_count    per detection row: kept-candidate count per (category, image); per GT row: non-ignored GTs per (category, area)
//   k_eval_clamp    count -> min(count, 100) (maxDets)
//   scan_exclusive  -> base[c * n + i]: the (category, image, score rank) layout of every kept detection
//   k_eval_match    one warp per (image, category): stable score rank, fp64 bbIou, greedy matching for 4 areas x 10 IoU thresholds
//   radix sort      stable LSD sort of the kept detections by (category, descending score); ties keep the (image, rank) layout
//   k_acc_tiles / k_acc_scan / k_acc_prec / k_acc_final
//                   per (category, area, threshold): cumulative tp / fp, precision at every true positive, the right-to-left max
//                   envelope sampled at the 101 recall thresholds
#include "common.cuh"

#define EV_MAXDET 100
#define EV_T 10
#define EV_A 4
#define EV_R 101
#define EV_WARPS 4                 // match kernel: warps per CTA
#define EV_IOU_CAP 800             // match kernel: fp64 IoU entries staged per warp (fast path: ng <= 32, kept * ng <= cap)
#define RS_THREADS 256
#define RS_ITEMS 8
#define RS_TILE (RS_THREADS * RS_ITEMS)
#define AC_THREADS 256
#define AC_ITEMS 8
#define AC_TILE (AC_THREADS * AC_ITEMS)

// order of np.argsort(-score, kind='mergesort') as an unsigned key (ascending key = descending score): -0 sorts with +0,
// NaN last; equal keys keep input order because every sort below is stable.
__device__ __forceinline__ uint32_t ev_score_key(float s)
{
    if (s != s) return 0xffffffffu;
    if (s == 0.f) s = 0.f;
    uint32_t u = __float_as_uint(s);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ~u;
}

struct EvBox { float x, y, w, h, area; };

// _to_prophesee: x = x1, y = y1, w = x2 - x1, h = y2 - y1 in float32; loadRes / _to_coco_format: area = w * h in float32
__device__ __forceinline__ EvBox ev_box(const float *__restrict__ b, int64_t r)
{
    const float4 v = __ldg(reinterpret_cast<const float4 *>(b) + r);
    EvBox o;
    o.x = v.x; o.y = v.y; o.w = __fsub_rn(v.z, v.x); o.h = __fsub_rn(v.w, v.y); o.area = __fmul_rn(o.w, o.h);
    return o;
}

// pycocotools maskApi.c bbIou (iscrowd = 0), in double, no contraction
__device__ __forceinline__ double ev_iou(const EvBox &d, const EvBox &g)
{
    const double dx = d.x, dy = d.y, dw = d.w, dh = d.h, gx = g.x, gy = g.y, gw = g.w, gh = g.h;
    const double w = __dsub_rn(fmin(__dadd_rn(dw, dx), __dadd_rn(gw, gx)), fmax(dx, gx));
    if (w <= 0) return 0.0;
    const double h = __dsub_rn(fmin(__dadd_rn(dh, dy), __dadd_rn(gh, gy)), fmax(dy, gy));
    if (h <= 0) return 0.0;
    const double i = __dmul_rn(w, h);
    const double u = __dsub_rn(__dadd_rn(__dmul_rn(dw, dh), __dmul_rn(gw, gh)), i);
    return __ddiv_rn(i, u);
}

__device__ __forceinline__ bool ev_out(float area, const dagr_eval_params_t &p, int a)
{
    const double v = area;
    return v < p.area_rng[a][0] || v > p.area_rng[a][1];
}

__device__ __forceinline__ int64_t ev_image_of(const int64_t *__restrict__ off, int64_t n, int64_t row)
{
    int64_t lo = 0, hi = n;                                              // last i with off[i] <= row
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(off + mid) <= row) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void k_eval_count(const int64_t *__restrict__ gt_label, const float *__restrict__ gt_box, const int64_t *__restrict__ gt_off,
                             const int64_t *__restrict__ dt_label, const int64_t *__restrict__ dt_off, int64_t n, int K, int64_t G,
                             int64_t D, const dagr_eval_params_t p, int *__restrict__ cnt, int *__restrict__ npig)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < D) {
        const uint32_t c = (uint32_t)__ldg(dt_label + r);
        const int64_t i = ev_image_of(dt_off, n, r);
        if (c < (uint32_t)K && __ldg(gt_off + i + 1) > __ldg(gt_off + i)) atomicAdd(cnt + (int64_t)c * n + i, 1);
    }
    if (r < G) {
        const uint32_t c = (uint32_t)__ldg(gt_label + r);
        if (c < (uint32_t)K) {
            const float area = ev_box(gt_box, r).area;
            for (int a = 0; a < EV_A; a++)
                if (!ev_out(area, p, a)) atomicAdd(npig + c * EV_A + a, 1);
        }
    }
}

__global__ void k_eval_clamp(int *__restrict__ cnt, int64_t m)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) cnt[i] = min(cnt[i], EV_MAXDET);
}

struct EvWarpSmem {
    EvBox det[EV_MAXDET];
    uint32_t key[EV_MAXDET];
    uint32_t flags[EV_MAXDET][EV_A];           // bits 0..9: true positive at threshold t, bits 16..25: false positive
    EvBox gt[32];
    double iou[EV_IOU_CAP];
};

// evaluateImg for one (area, threshold) combination over the kept detections of one (image, category).  FAST: the class's
// GTs (ng <= 32) and their IoU table are staged, the matched set is a register mask; otherwise the GTs are read from the
// image's rows, the IoU is recomputed (same function, same bits) and the matched set lives in gtm[row] (bit = combination).
template <bool FAST>
__device__ void ev_match_combo(EvWarpSmem &s, int nk, int ng, int cmb, const dagr_eval_params_t &p, const float *__restrict__ gt_box,
                               const int64_t *__restrict__ gt_label, int64_t g0, int64_t g1, uint32_t c,
                               unsigned long long *__restrict__ gtm)
{
    const int a = cmb / EV_T, t = cmb % EV_T;
    uint32_t mask = 0;
    for (int d = 0; d < nk; d++) {
        const double thr0 = fmin(p.iou_thrs[t], 1.0 - 1e-10);
        double best = thr0;
        int64_t m = -1;
        bool mig = false;
        // pass 0: the GTs inside the area range in input order, pass 1 (only if pass 0 found none): the ignored ones
        // (evaluateImg's stable ignore-last order with its `break`)
        for (int pass = 0; pass < 2 && m < 0; pass++) {
            if (FAST) {
                for (int g = 0; g < ng; g++) {
                    if (ev_out(s.gt[g].area, p, a) != (pass == 1) || ((mask >> g) & 1u)) continue;
                    const double v = s.iou[d * ng + g];
                    if (v < best) continue;
                    best = v; m = g;
                }
            } else {
                for (int64_t g = g0; g < g1; g++) {
                    if ((uint32_t)__ldg(gt_label + g) != c) continue;
                    const EvBox gb = ev_box(gt_box, g);
                    if (ev_out(gb.area, p, a) != (pass == 1) || ((gtm[g] >> cmb) & 1ull)) continue;
                    const double v = ev_iou(s.det[d], gb);
                    if (v < best) continue;
                    best = v; m = g;
                }
            }
            mig = pass == 1;
        }
        bool tp = false, ig;
        if (m >= 0) {
            if (FAST) mask |= 1u << m; else atomicOr(gtm + m, 1ull << cmb);
            tp = !mig; ig = mig;
        } else {
            ig = ev_out(s.det[d].area, p, a);
        }
        if (!ig) atomicOr(&s.flags[d][a], tp ? (1u << t) : (1u << (16 + t)));
    }
}

__global__ void __launch_bounds__(EV_WARPS * 32) k_eval_match(
    const float *__restrict__ gt_box, const int64_t *__restrict__ gt_label, const int64_t *__restrict__ gt_off,
    const float *__restrict__ dt_box, const float *__restrict__ dt_score, const int64_t *__restrict__ dt_label,
    const int64_t *__restrict__ dt_off, int64_t n, int K, const dagr_eval_params_t p, const int *__restrict__ kept,
    const int *__restrict__ base, unsigned long long *__restrict__ keys, uint32_t *__restrict__ vals, uint32_t *__restrict__ flags,
    unsigned long long *__restrict__ gtm)
{
    __shared__ EvWarpSmem sm[EV_WARPS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * EV_WARPS + wid;
    if (gw >= n * K) return;
    const int64_t i = gw / K;
    const uint32_t c = (uint32_t)(gw % K);
    const int nk = kept[(int64_t)c * n + i];
    if (nk == 0) return;
    EvWarpSmem &s = sm[wid];
    const int b0 = base[(int64_t)c * n + i];
    const int64_t d0 = dt_off[i], d1 = dt_off[i + 1], g0 = gt_off[i], g1 = gt_off[i + 1];

    // stable rank of each detection of class c by descending score; the first 100 are kept, in rank order
    for (int64_t j0 = d0; j0 < d1; j0 += 32) {
        const int64_t j = j0 + lane;
        const bool mine = j < d1 && (uint32_t)__ldg(dt_label + j) == c;
        const uint32_t kj = mine ? ev_score_key(__ldg(dt_score + j)) : 0u;
        int rank = 0;
        for (int64_t k = d0; k < d1; k++) {
            if ((uint32_t)__ldg(dt_label + k) != c) continue;
            const uint32_t kk = ev_score_key(__ldg(dt_score + k));
            rank += kk < kj || (kk == kj && k < j);
        }
        if (mine && rank < EV_MAXDET) { s.det[rank] = ev_box(dt_box, j); s.key[rank] = kj; }
    }
    for (int d = lane; d < nk; d += 32)
#pragma unroll
        for (int a = 0; a < EV_A; a++) s.flags[d][a] = 0;

    // the class's GTs of this image in input order
    int ng = 0;
    for (int64_t g = g0; g < g1; g += 32) {
        const bool mine = g + lane < g1 && (uint32_t)__ldg(gt_label + g + lane) == c;
        const unsigned bal = __ballot_sync(0xffffffffu, mine);
        const int at = ng + __popc(bal & ((1u << lane) - 1u));
        if (mine && at < 32) s.gt[at] = ev_box(gt_box, g + lane);
        if (mine) gtm[g + lane] = 0ull;
        ng += __popc(bal);
    }
    __syncwarp();
    const bool fast = ng <= 32 && nk * ng <= EV_IOU_CAP;
    if (fast)
        for (int e = lane; e < nk * ng; e += 32) s.iou[e] = ev_iou(s.det[e / ng], s.gt[e % ng]);
    __syncwarp();

    for (int cmb = lane; cmb < EV_A * EV_T; cmb += 32) {
        if (fast) ev_match_combo<true>(s, nk, ng, cmb, p, gt_box, gt_label, g0, g1, c, gtm);
        else ev_match_combo<false>(s, nk, ng, cmb, p, gt_box, gt_label, g0, g1, c, gtm);
    }
    __syncwarp();
    for (int d = lane; d < nk; d += 32) {
        const int o = b0 + d;
        keys[o] = ((unsigned long long)c << 32) | s.key[d];
        vals[o] = (uint32_t)o;
        reinterpret_cast<uint4 *>(flags)[o] = make_uint4(s.flags[d][0], s.flags[d][1], s.flags[d][2], s.flags[d][3]);
    }
}

// ---- stable LSD radix sort of (key u64, val u32) pairs, 8 bits per pass, *count items read on the device --------------
__global__ void __launch_bounds__(RS_THREADS) k_rs_hist(const unsigned long long *__restrict__ keys, const int *__restrict__ count,
                                                        int shift, int ntiles, int *__restrict__ hist)
{
    __shared__ int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int64_t m = *count, t0 = (int64_t)blockIdx.x * RS_TILE;
    for (int k = 0; k < RS_ITEMS; k++) {
        const int64_t e = t0 + k * RS_THREADS + threadIdx.x;
        if (e < m) atomicAdd(&h[(int)((keys[e] >> shift) & 255ull)], 1);
    }
    __syncthreads();
    hist[(int64_t)threadIdx.x * ntiles + blockIdx.x] = h[threadIdx.x];
}

__global__ void __launch_bounds__(RS_THREADS) k_rs_scatter(const unsigned long long *__restrict__ kin, const uint32_t *__restrict__ vin,
                                                           const int *__restrict__ count, int shift, int ntiles,
                                                           const int *__restrict__ off, unsigned long long *__restrict__ kout,
                                                           uint32_t *__restrict__ vout)
{
    __shared__ int run[256];
    __shared__ int wc[RS_THREADS / 32][256];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t m = *count, t0 = (int64_t)blockIdx.x * RS_TILE;
    if (t0 >= m) return;
    run[threadIdx.x] = off[(int64_t)threadIdx.x * ntiles + blockIdx.x];
    for (int w = 0; w < RS_THREADS / 32; w++) wc[w][threadIdx.x] = 0;
    __syncthreads();
    for (int k = 0; k < RS_ITEMS; k++) {
        const int64_t e = t0 + k * RS_THREADS + threadIdx.x;
        const bool live = e < m;
        unsigned long long key = 0; uint32_t val = 0;
        if (live) { key = kin[e]; val = vin[e]; }
        const int dg = live ? (int)((key >> shift) & 255ull) : 256;
        const unsigned peers = __match_any_sync(0xffffffffu, dg);
        const int rk = __popc(peers & ((1u << lane) - 1u));
        if (live && rk == 0) wc[wid][dg] = __popc(peers);
        __syncthreads();
        {                                                                // per digit: exclusive offsets of the warps, in order
            int r = run[threadIdx.x];
            for (int w = 0; w < RS_THREADS / 32; w++) { const int v = wc[w][threadIdx.x]; wc[w][threadIdx.x] = r; r += v; }
            run[threadIdx.x] = r;
        }
        __syncthreads();
        if (live) { const int o = wc[wid][dg] + rk; kout[o] = key; vout[o] = val; }
        __syncthreads();
        for (int w = 0; w < RS_THREADS / 32; w++) wc[w][threadIdx.x] = 0;
        __syncthreads();
    }
}

// ---- accumulate ------------------------------------------------------------------------------------------------------
// tile-local counts of one (category, area): per threshold, true positives in the low 16 bits and false positives in the high
__device__ __forceinline__ void ac_counts(const uint32_t *__restrict__ flags, const uint32_t *__restrict__ vals, int64_t s, int64_t e,
                                          int64_t first, int a, uint32_t f[AC_ITEMS], int cntv[EV_T])
{
#pragma unroll
    for (int k = 0; k < AC_ITEMS; k++) {
        const int64_t x = first + k;
        f[k] = x < e ? __ldg(flags + (int64_t)__ldg(vals + s + x) * EV_A + a) : 0u;
    }
#pragma unroll
    for (int t = 0; t < EV_T; t++) {
        int v = 0;
#pragma unroll
        for (int k = 0; k < AC_ITEMS; k++) v += ((f[k] >> t) & 1u) | (((f[k] >> (16 + t)) & 1u) << 16);
        cntv[t] = v;
    }
}

__global__ void __launch_bounds__(AC_THREADS) k_acc_tiles(const uint32_t *__restrict__ flags, const uint32_t *__restrict__ vals,
                                                          const int *__restrict__ base, int64_t n, int ntmax,
                                                          int *__restrict__ tile_tot)
{
    __shared__ int sm[32];
    __shared__ int tot;
    const int c = blockIdx.z, a = blockIdx.y;
    const int64_t s = base[(int64_t)c * n], L = base[(int64_t)(c + 1) * n] - s;
    if ((int64_t)blockIdx.x * AC_TILE >= L) return;
    uint32_t f[AC_ITEMS];
    int cntv[EV_T];
    ac_counts(flags, vals, s, L, (int64_t)blockIdx.x * AC_TILE + (int64_t)threadIdx.x * AC_ITEMS, a, f, cntv);
    for (int t = 0; t < EV_T; t++) {
        block_exclusive_scan(cntv[t], &tot, sm);
        if (threadIdx.x == 0) tile_tot[(((int64_t)c * EV_A + a) * ntmax + blockIdx.x) * EV_T + t] = tot;
        __syncthreads();
    }
}

// one thread per (category, area, threshold): exclusive prefix of the tile counts (tp, fp as two int32 words)
__global__ void k_acc_scan(const int *__restrict__ tile_tot, const int *__restrict__ base, int64_t n, int K, int ntmax,
                           int2 *__restrict__ tile_pre, int2 *__restrict__ total)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= K * EV_A * EV_T) return;
    const int c = q / (EV_A * EV_T), a = (q / EV_T) % EV_A, t = q % EV_T;
    const int64_t L = base[(int64_t)(c + 1) * n] - base[(int64_t)c * n];
    const int nt = (int)((L + AC_TILE - 1) / AC_TILE);
    int tp = 0, fp = 0;
    for (int x = 0; x < nt; x++) {
        const int64_t o = ((int64_t)c * EV_A + a) * ntmax + x;
        tile_pre[o * EV_T + t] = make_int2(tp, fp);
        const int v = tile_tot[o * EV_T + t];
        tp += v & 0xffff; fp += v >> 16;
    }
    total[q] = make_int2(tp, fp);
}

// per true positive j (1-based) with fp false positives before it: pr = j / (fp + j + eps), rc = j / npig; pr is a candidate
// of q[r] for every recall threshold r with rec_thrs[r] <= rc.  bucket[R] = max pr over the true positives whose largest
// such r is R (a suffix max over the buckets then gives the envelope at searchsorted(rc, rec_thrs, 'left')).
__global__ void __launch_bounds__(AC_THREADS) k_acc_prec(const uint32_t *__restrict__ flags, const uint32_t *__restrict__ vals,
                                                         const int *__restrict__ base, int64_t n, int ntmax,
                                                         const int *__restrict__ npig, const int2 *__restrict__ tile_pre,
                                                         const dagr_eval_params_t p, unsigned long long *__restrict__ bucket)
{
    __shared__ int sm[32];
    __shared__ int tot;
    __shared__ unsigned long long bk[EV_T][EV_R];
    const int c = blockIdx.z, a = blockIdx.y;
    const int64_t s = base[(int64_t)c * n], L = base[(int64_t)(c + 1) * n] - s;
    const int np = npig[c * EV_A + a];
    if ((int64_t)blockIdx.x * AC_TILE >= L || np == 0) return;
    for (int e = threadIdx.x; e < EV_T * EV_R; e += AC_THREADS) (&bk[0][0])[e] = 0ull;
    uint32_t f[AC_ITEMS];
    int cntv[EV_T];
    ac_counts(flags, vals, s, L, (int64_t)blockIdx.x * AC_TILE + (int64_t)threadIdx.x * AC_ITEMS, a, f, cntv);
    const double eps = 0x1p-52;                                         // np.spacing(1)
    for (int t = 0; t < EV_T; t++) {
        const int ex = block_exclusive_scan(cntv[t], &tot, sm);
        const int2 pre = tile_pre[(((int64_t)c * EV_A + a) * ntmax + blockIdx.x) * EV_T + t];
        int tp = pre.x + (ex & 0xffff), fp = pre.y + (ex >> 16);
        int curR = -1;
        unsigned long long cur = 0ull;
#pragma unroll
        for (int k = 0; k < AC_ITEMS; k++) {
            if ((f[k] >> (16 + t)) & 1u) fp++;
            if (!((f[k] >> t) & 1u)) continue;
            tp++;
            const double dtp = (double)tp;
            const double pr = __ddiv_rn(dtp, __dadd_rn(__dadd_rn((double)fp, dtp), eps));
            const double rc = __ddiv_rn(dtp, (double)np);
            int lo = 0, hi = EV_R;                                       // R = (number of rec_thrs <= rc) - 1
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (p.rec_thrs[mid] <= rc) lo = mid + 1; else hi = mid; }
            const int R = lo - 1;
            const unsigned long long b = (unsigned long long)__double_as_longlong(pr);
            if (R != curR) { if (curR >= 0) atomicMax(&bk[t][curR], cur); curR = R; cur = b; }
            else cur = cur > b ? cur : b;
        }
        if (curR >= 0) atomicMax(&bk[t][curR], cur);
    }
    __syncthreads();
    unsigned long long *gb = bucket + ((int64_t)c * EV_A + a) * EV_T * EV_R;
    for (int e = threadIdx.x; e < EV_T * EV_R; e += AC_THREADS) {
        const unsigned long long v = (&bk[0][0])[e];
        if (v) atomicMax(gb + e, v);
    }
}

__global__ void k_acc_final(const unsigned long long *__restrict__ bucket, const int *__restrict__ npig, const int2 *__restrict__ total,
                            const int *__restrict__ base, int64_t n, int K, double *__restrict__ precision, double *__restrict__ recall)
{
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= K * EV_A * EV_T) return;
    const int c = q / (EV_A * EV_T), a = (q / EV_T) % EV_A, t = q % EV_T;
    const int np = npig[c * EV_A + a];
    const int64_t nd = base[(int64_t)(c + 1) * n] - base[(int64_t)c * n];
    const unsigned long long *b = bucket + (int64_t)q * EV_R;
    unsigned long long mx = 0ull;
    for (int r = EV_R - 1; r >= 0; r--) {
        mx = mx > b[r] ? mx : b[r];
        precision[(((int64_t)t * EV_R + r) * K + c) * EV_A + a] = np == 0 ? -1.0 : __longlong_as_double((long long)mx);
    }
    recall[((int64_t)t * K + c) * EV_A + a] = np == 0 ? -1.0 : nd == 0 ? 0.0 : __ddiv_rn((double)total[q].x, (double)np);
}

// ---- C-ABI ------------------------------------------------------------------------------------------------------------
struct EvLayout {
    int64_t cnt, base, blocksums, npig, keys0, keys1, vals0, vals1, flags, gtm, rs_hist, tile_tot, tile_pre, total, bucket, bytes;
    int rs_tiles, ac_tiles, rs_bits;
};

static int ev_bits(int64_t v) { int b = 0; while ((1ll << b) < v) b++; return b; }
static int64_t ev_align(int64_t v) { return (v + 255) & ~(int64_t)255; }

static EvLayout ev_layout(int64_t n, int K, int64_t G, int64_t D)
{
    EvLayout L;
    const int64_t nk = n * K, m = D > 0 ? D : 1;
    L.rs_tiles = (int)((m + RS_TILE - 1) / RS_TILE);
    const int64_t per_cat = D < n * EV_MAXDET ? D : n * EV_MAXDET;
    L.ac_tiles = (int)((per_cat + AC_TILE - 1) / AC_TILE) + 1;
    L.rs_bits = 32 + ev_bits(K);
    const int64_t nscan = nk + 1 > 256ll * L.rs_tiles ? nk + 1 : 256ll * L.rs_tiles;
    int64_t o = 0;
    auto take = [&](int64_t bytes) { const int64_t at = o; o += ev_align(bytes); return at; };
    L.cnt = take(4 * (nk + 1));
    L.base = take(4 * (nk + 1));
    L.blocksums = take(4 * (dagr_scan_blocks(nscan) + 2));
    L.npig = take(4ll * K * EV_A);
    L.keys0 = take(8 * m); L.keys1 = take(8 * m);
    L.vals0 = take(4 * m); L.vals1 = take(4 * m);
    L.flags = take(16 * m);
    L.gtm = take(8 * (G > 0 ? G : 1));
    L.rs_hist = take(4 * (256ll * L.rs_tiles + 1));
    L.tile_tot = take(4ll * K * EV_A * L.ac_tiles * EV_T);
    L.tile_pre = take(8ll * K * EV_A * L.ac_tiles * EV_T);
    L.total = take(8ll * K * EV_A * EV_T);
    L.bucket = take(8ll * K * EV_A * EV_T * EV_R);
    L.bytes = o;
    return L;
}

static bool ev_shape_ok(int64_t n, int K, int64_t G, int64_t D)
{
    return n >= 1 && K >= 1 && G >= 0 && D >= 0 && n * K < (1ll << 31) - 1 && D < (1ll << 31) && G < (1ll << 40) &&
           K <= 65535 && n < (1ll << 31) / EV_MAXDET;
}

extern "C" int dagr_eval_workspace_bytes(int64_t n_images, int K, int64_t n_gt, int64_t n_det, int64_t *bytes)
{
    DAGR_CHECK_ARG(bytes != nullptr, "null bytes");
    DAGR_CHECK_ARG(ev_shape_ok(n_images, K, n_gt, n_det), "n_images >= 1, K in [1, 65535], n_images * K < 2^31 - 1, "
                   "n_det < 2^31 and n_images < 2^31 / 100");
    *bytes = ev_layout(n_images, K, n_gt, n_det).bytes;
    return DAGR_OK;
}

extern "C" int dagr_evaluate_bbox(const float *gt_box, const int64_t *gt_label, const int64_t *gt_off, const float *dt_box,
                                  const float *dt_score, const int64_t *dt_label, const int64_t *dt_off, int64_t n_images, int K,
                                  int64_t n_gt, int64_t n_det, const dagr_eval_params_t *params_host, void *workspace,
                                  int64_t workspace_bytes, double *precision, double *recall, void *stream)
{
    DAGR_CHECK_ARG(params_host && gt_off && dt_off && workspace && precision && recall, "null pointer");
    DAGR_CHECK_ARG(ev_shape_ok(n_images, K, n_gt, n_det), "n_images >= 1, K in [1, 65535], n_images * K < 2^31 - 1, "
                   "n_det < 2^31 and n_images < 2^31 / 100");
    DAGR_CHECK_ARG(n_gt == 0 || (gt_box && gt_label), "null GT rows");
    DAGR_CHECK_ARG(n_det == 0 || (dt_box && dt_score && dt_label), "null detection rows");
    DAGR_CHECK_ARG(((uintptr_t)gt_box & 15) == 0 && ((uintptr_t)dt_box & 15) == 0, "boxes must be 16-byte aligned");
    const EvLayout L = ev_layout(n_images, K, n_gt, n_det);
    DAGR_CHECK_ARG(workspace_bytes >= L.bytes && ((uintptr_t)workspace & 255) == 0,
                   "workspace smaller than dagr_eval_workspace_bytes or not 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    char *w = (char *)workspace;
    int *cnt = (int *)(w + L.cnt), *base = (int *)(w + L.base), *bs = (int *)(w + L.blocksums), *npig = (int *)(w + L.npig);
    unsigned long long *keys[2] = {(unsigned long long *)(w + L.keys0), (unsigned long long *)(w + L.keys1)};
    uint32_t *vals[2] = {(uint32_t *)(w + L.vals0), (uint32_t *)(w + L.vals1)};
    uint32_t *flags = (uint32_t *)(w + L.flags);
    int *hist = (int *)(w + L.rs_hist), *tile_tot = (int *)(w + L.tile_tot);
    int2 *tile_pre = (int2 *)(w + L.tile_pre), *total = (int2 *)(w + L.total);
    unsigned long long *bucket = (unsigned long long *)(w + L.bucket), *gtm = (unsigned long long *)(w + L.gtm);
    const int64_t nk = n_images * K;
    const dagr_eval_params_t p = *params_host;

    DAGR_CUDA(cudaMemsetAsync(cnt, 0, 4 * nk, st));
    DAGR_CUDA(cudaMemsetAsync(npig, 0, 4ll * K * EV_A, st));
    DAGR_CUDA(cudaMemsetAsync(bucket, 0, 8ll * K * EV_A * EV_T * EV_R, st));
    const int64_t rows = n_gt > n_det ? n_gt : n_det;
    if (rows > 0)
        k_eval_count<<<dagr_div_up(rows, 256), 256, 0, st>>>(gt_label, gt_box, gt_off, dt_label, dt_off, n_images, K, n_gt, n_det, p,
                                                             cnt, npig);
    k_eval_clamp<<<dagr_div_up(nk, 256), 256, 0, st>>>(cnt, nk);
    scan_exclusive(cnt, base, nk, bs, st);                             // base[nk] = kept detections in all
    DAGR_CHECK_LAUNCH();
    k_eval_match<<<dagr_div_up(nk, EV_WARPS), EV_WARPS * 32, 0, st>>>(gt_box, gt_label, gt_off, dt_box, dt_score, dt_label, dt_off,
                                                                      n_images, K, p, cnt, base, keys[0], vals[0], flags, gtm);
    DAGR_CHECK_LAUNCH();
    int cur = 0;
    for (int shift = 0; shift < L.rs_bits; shift += 8, cur ^= 1) {
        k_rs_hist<<<L.rs_tiles, RS_THREADS, 0, st>>>(keys[cur], base + nk, shift, L.rs_tiles, hist);
        scan_exclusive(hist, hist, 256ll * L.rs_tiles, bs, st);
        k_rs_scatter<<<L.rs_tiles, RS_THREADS, 0, st>>>(keys[cur], vals[cur], base + nk, shift, L.rs_tiles, hist, keys[cur ^ 1],
                                                        vals[cur ^ 1]);
        DAGR_CHECK_LAUNCH();
    }
    const dim3 g(L.ac_tiles, EV_A, K);
    k_acc_tiles<<<g, AC_THREADS, 0, st>>>(flags, vals[cur], base, n_images, L.ac_tiles, tile_tot);
    const int nq = K * EV_A * EV_T;
    k_acc_scan<<<dagr_div_up(nq, 128), 128, 0, st>>>(tile_tot, base, n_images, K, L.ac_tiles, tile_pre, total);
    k_acc_prec<<<g, AC_THREADS, 0, st>>>(flags, vals[cur], base, n_images, L.ac_tiles, npig, tile_pre, p, bucket);
    k_acc_final<<<dagr_div_up(nq, 128), 128, 0, st>>>(bucket, npig, total, base, n_images, K, precision, recall);
    DAGR_CHECK_LAUNCH();
    return DAGR_OK;
}
