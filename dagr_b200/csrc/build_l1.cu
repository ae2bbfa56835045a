// build_l1.cu -- fused event-level build: spiral probe on a shared-memory hashed grid + conv_a.
//
// One CTA per pool1 voxel.  Because events are stored in cell-major order, the voxel's own events are
// one contiguous range and the events of its 3x3 voxel neighbourhood are THREE contiguous runs (one per
// voxel row), so the (t, arrival idx, polarity) records the probe needs are staged in shared memory
// with fully coalesced loads.  A per-tile-pixel bin table (shared memory) maps each of the
// (CW+2r) x (CH+2r) pixels the voxel's events can reach to its FIFO column (newest <= Q entries,
// ev_graph.cu:201-211).  The spiral probe (ev_graph.cu:49-78) then runs entirely on chip; accepted
// neighbours are written to the column-major ELL and folded into conv_block1.conv_block1 on the fly
// (their features are (polarity, x/W, y/H): no gather at all).
// Voxels whose neighbourhood does not fit the staging buffer fall back to probing global memory.
#include <type_traits>
#include "common.cuh"

// Two instances of the per-voxel routine (template parameters CAP = staged neighbourhood records, THREADS = CTA size):
//   regular : one CTA per pool1 voxel, 160 threads (>= events of a voxel at the nominal density, Poisson mean 134: one
//             pass), 2048 staged records, 4 CTAs per SM -- or, while no dense voxels are expected (defer = 0), the lean
//             launch with 1536 records (uniform 300k events/sample need ~1200-1450) and 5 CTAs per SM: the kernel is
//             latency bound, 25 instead of 20 warps per SM make it faster;
//   dense   : voxels whose 3x3 neighbourhood holds more records than that (moving edges in real / clustered streams: 58 %
//             of the events of the clustered benchmark stream) are pushed on a device work list by the regular kernel and
//             processed by a persistent second kernel (one 512-thread CTA per SM, 12288 staged records, dynamic pop) --
//             the global-memory probe remains only as the fallback behind that.
#define BL_THREADS 160
#define BL_CAP 2048
#define BL_CAP_LEAN 1536           // the count-only launch (defer = 0): 44 KB per CTA -> five CTAs per SM instead of four
#define BL_THREADS_BIG 512
#define BL_CAP_BIG 12288
#define BL_NB 8                  // time buckets of width delta_t kept per tile pixel

struct BLTile {
    int X0, Y0, TW, TH;          // tile origin (pixel) and extent
    int run_start[3], run_off[3], run_len[3];
    int smin, smax;              // slice (t / delta_t) range of the voxel's own events
    int unsorted;                // some pixel's records are not time-sorted -> no time bucketing
    int bucketed;                // the bucket ranges are in use (kept here, not in a register live through the event loop)
    int maxidx;                  // newest arrival index among the events this launch must process (-1: none)
};

__host__ __device__ __forceinline__ size_t bl_acc_offset(const dagr_geom_t &g, int cap)
{
    const size_t TW = g.CW + 2 * g.r, TH = g.CH + 2 * g.r, TP = TW * TH;
    const size_t o = (size_t)(2 * g.r + 1) * 32 + (size_t)cap * 12 + TP * 4 + (TW + TH) * 4 + TP * BL_NB * 2 + (size_t)g.ncell * 4;
    return (o + 15) / 16 * 16;
}
// The occupancy masks are built only for the ring walk and s_order only serves the cell walk, so the two share one region.
// The cell walk runs when a tile side exceeds 32 px or r > 8; then TWmax + THmax >= 33 and the masks' region is the larger one.
static size_t bl_smem_bytes(const dagr_geom_t *g, int cap, int threads)
{
    const size_t TW = g->CW + 2 * g->r, TH = g->CH + 2 * g->r;
    const size_t occ = (size_t)BL_NB * (TW + TH) * 4, order = (size_t)threads * 2;
    return bl_acc_offset(*g, cap) + (size_t)(DAGR_ELL - 1) * threads * 4 + (occ > order ? occ : order) + 16;
}

#define BL_R1 96                 // spiral cells walked one-thread-per-event before unsaturated events are handed
                                 // to the warp-cooperative continuation (saturated events need ~85 cells)

// Phase 1: warp-converged probe.  All lanes walk the spiral in lock step (same cell index c), four cells per
// iteration so the dependent shared-memory loads pipeline; the per-bin record loop runs to the warp-wide
// maximum with predication and the walk ends when every lane has its K-1 neighbours.  Lanes of a warp are
// events of similar age (threads are assigned in arrival order) and each tile pixel exposes only the
// sub-range of its FIFO column that can lie within delta_t of the event (time buckets), so the common
// iteration touches no record at all.
template <bool STAGED, int THREADS>
__device__ __forceinline__ void bl_probe(const dagr_geom_t &g, int64_t N, int p, bool active, const int2 me, int eb, int tidx0,
                                         int c_end, const uint32_t *s_pbin, const uint16_t *s_rng, const short *s_sp2,
                                         const int2 *s_ti, const int2 *__restrict__ ti, uint32_t *s_acc,
                                         int32_t *__restrict__ nbr, uint16_t *__restrict__ off, int &n_out)
{
    const int kmax = g.K - 1;
    int n = active ? 0 : kmax;
    for (int c0 = 0; c0 < c_end; c0 += 4) {
        if (__all_sync(0xffffffffu, n >= kmax)) break;
        uint32_t rg[4]; int pix[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int c = min(c0 + u, g.ncell - 1);
            pix[u] = tidx0 + s_sp2[c];
        }
#pragma unroll
        for (int u = 0; u < 4; u++) rg[u] = s_rng[pix[u] * BL_NB + eb];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int c = c0 + u;
            const int lo = rg[u] & 0xff, hi = rg[u] >> 8;
            const int cnt = (c < c_end && n < kmax) ? hi - lo : 0;
            if (!__any_sync(0xffffffffu, cnt > 0)) continue;
            const int base = (int)(s_pbin[pix[u]] >> 8);
            const int vmax = __reduce_max_sync(0xffffffffu, cnt);
            for (int k = 0; k < vmax; k++) {
                if (k < cnt && n < kmax) {
                    // FIFO order: newest first.  Visible records of the pixel are [base, base+vis) in arrival order;
                    // the bucket range [lo,hi) counts from the OLDEST visible record.
                    const int j = base + hi - 1 - k;
                    const int2 o = STAGED ? s_ti[j] : __ldg(ti + j);
                    if (o.y < me.y && me.x - o.x <= g.dt_us) {              // ev_graph.cu:64-69
                        // accepted (record, cell) pairs wait in shared memory for phase B (staged mode)
                        if (STAGED) s_acc[n * THREADS + threadIdx.x] = ((uint32_t)j << 10) | (uint32_t)c;
                        else { nbr[(int64_t)n * N + p] = j; off[(int64_t)n * N + p] = (uint16_t)c; }
                        n++;
                    }
                }
            }
        }
    }
    n_out = active ? n : 0;
}


#ifndef BL_SHARED_ADDR
#define BL_SHARED_ADDR 1
#endif
// explicit 32-bit shared-memory accesses for the ring walk: with generic pointers ptxas re-materialises the shared window base
// (S2R SR_CgaCtaId + MOV + LEA) inside the pop loop instead of keeping it in a register (slower in an A/B).
// The same treatment of phase B's seven table bases (the conv_a accumulation loop) costs registers the 45 accumulators do not
// leave (stack 16 -> 40 bytes, slower) -- that loop keeps its generic pointers.
__device__ __forceinline__ uint32_t bl_sa(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t bl_lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint32_t bl_lds16(uint32_t a) { uint32_t v; asm volatile("{ .reg .u16 t; ld.shared.u16 t, [%1]; cvt.u32.u16 %0, t; }" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ int bl_lds16s(uint32_t a) { int v; asm volatile("{ .reg .s16 t; ld.shared.s16 t, [%1]; cvt.s32.s16 %0, t; }" : "=r"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ int2 bl_lds64(uint32_t a) { int2 v; asm volatile("ld.shared.v2.s32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory"); return v; }
#ifndef BL_FAST_TABLES
#define BL_FAST_TABLES 1            // exact reciprocal division for the time buckets (faster in an A/B)
#endif
// t / d for 0 <= t < 2^24 through a float reciprocal and one exact fix-up step (the generic 32-bit division is ~20 instructions);
// anything else takes the plain division, so the result is always the C quotient
__device__ __forceinline__ int bl_div(int t, int d, float inv)
{
#if BL_FAST_TABLES
    if ((unsigned)t >= (1u << 24)) return t / d;
    int q = (int)((float)t * inv);
    const int r = t - q * d;
    if (r < 0) q--; else if (r >= d) q++;
    return q;
#else
    (void)inv;
    return t / d;
#endif
}
__device__ __forceinline__ void bl_sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }

// Ring walk with occupancy bitmasks.  For every time bucket e the CTA keeps, per tile row, a 32-bit mask of the
// pixels whose bucket range is non-empty (and the transposed per-column masks).  Ring d of the spiral consists of
// four straight segments (spiral.h: right column upwards, top row leftwards, left column downwards, bottom row
// rightwards, 2d cells each), so the candidate cells of a segment are one bit-field extract (+ a bit reversal
// for the two descending legs).  Each lane then visits ONLY its non-empty cells, in spiral order, by clearing
// the lowest set bit: empty pixels (~2/3 of the window) cost nothing and lanes are no longer held to the
// warp-wide maximum of per-cell work.  Unsaturated events simply run out of rings (no second phase needed).
template <bool STAGED, int THREADS>
__device__ __forceinline__ void bl_probe_rings(const dagr_geom_t &g, int64_t N, int p, bool active, const int2 me, int eb, int tx0, int ty0,
                                               int TW, int TH, const uint32_t *s_pbin, const uint16_t *s_rng, const uint32_t *s_occ_r,
                                               const uint32_t *s_occ_c, const short *s_sp2, const int2 *s_ti, const int2 *__restrict__ ti, uint32_t *s_acc,
                                               int32_t *__restrict__ nbr, uint16_t *__restrict__ off, int &n_out)
{
    const int kmax = g.K - 1;
    int n = active ? 0 : kmax;
    const uint32_t *occr = s_occ_r + eb * TH, *occc = s_occ_c + eb * TW;
    constexpr bool SA = STAGED && BL_SHARED_ADDR;
    const uint32_t a_rng = bl_sa(s_rng) + 2u * (uint32_t)eb, a_pbin = bl_sa(s_pbin), a_ti = bl_sa(s_ti), a_sp2 = bl_sa(s_sp2);
    const uint32_t a_acc = bl_sa(s_acc) + 4u * threadIdx.x;
    const int dt_us = g.dt_us;
    auto visit = [&](int pix, int c) {
        const uint32_t rg = SA ? bl_lds16(a_rng + (uint32_t)pix * (2u * BL_NB)) : (uint32_t)s_rng[pix * BL_NB + eb];
        const int lo = rg & 0xff, hi = rg >> 8;
        const int base = (int)((SA ? bl_lds32(a_pbin + 4u * (uint32_t)pix) : s_pbin[pix]) >> 8);
        for (int j = base + hi - 1; j >= base + lo && n < kmax; j--) {     // FIFO order: newest first
            const int2 o = SA ? bl_lds64(a_ti + 8u * (uint32_t)j) : (STAGED ? s_ti[j] : __ldg(ti + j));
            if (o.y < me.y && me.x - o.x <= dt_us) {                        // ev_graph.cu:64-69
                if (SA) bl_sts32(a_acc + (uint32_t)n * (4u * THREADS), ((uint32_t)j << 10) | (uint32_t)c);
                else if (STAGED) s_acc[n * THREADS + threadIdx.x] = ((uint32_t)j << 10) | (uint32_t)c;
                else { nbr[(int64_t)n * N + p] = j; off[(int64_t)n * N + p] = (uint16_t)c; }
                n++;
            }
        }
    };
    if (n < kmax && ((occr[ty0] >> tx0) & 1u)) visit(ty0 * TW + tx0, 0);   // spiral cell 0: own pixel
    const int tidx0 = ty0 * TW + tx0;
    for (int d = 1; d <= g.r; d++) {
        if (__all_sync(0xffffffffu, n >= kmax)) break;
        // one 8d-bit occupancy word per ring, bit i = spiral cell cbase + i (the four legs of spiral.h back to back), so a
        // lane runs ONE pop loop per ring instead of four: trip counts (popcount of a whole ring) vary much less between
        // the lanes of a warp than those of single legs
        const int l2 = 2 * d;
        const uint32_t fm = (l2 >= 32) ? 0xffffffffu : ((1u << l2) - 1u);
        const int cbase = (l2 - 1) * (l2 - 1);
        // the 8d mask bits live in two 32-bit words (d <= 8): bit i of `lo` = spiral cell cbase + i, of `hi` = cbase + 32 + i;
        // popping from a register pair costs a third of the 64-bit find-first-set / clear-lowest sequence
        uint32_t lo = 0, hi = 0;
        if (n < kmax) {
            const uint32_t leg0 = (occc[tx0 + d] >> (ty0 - d + 1)) & fm;                          // x = +d, y = -d+1 .. d
            const uint32_t leg1 = __brev((occr[ty0 + d] >> (tx0 - d)) & fm) >> (32 - l2);         // y = +d, x = d-1 .. -d
            const uint32_t leg2 = __brev((occc[tx0 - d] >> (ty0 - d)) & fm) >> (32 - l2);         // x = -d, y = d-1 .. -d
            const uint32_t leg3 = (occr[ty0 - d] >> (tx0 - d + 1)) & fm;                          // y = -d, x = -d+1 .. d
            const unsigned long long m = (unsigned long long)leg0 | ((unsigned long long)leg1 << l2) |
                                         ((unsigned long long)leg2 << (2 * l2)) | ((unsigned long long)leg3 << (3 * l2));
            lo = (uint32_t)m; hi = (uint32_t)(m >> 32);
        }
        while (lo | hi) {
            int i;
            if (lo) { i = __ffs((int)lo) - 1; lo &= lo - 1; }
            else    { i = 32 + __ffs((int)hi) - 1; hi &= hi - 1; }
            visit(tidx0 + (SA ? bl_lds16s(a_sp2 + 2u * (uint32_t)(cbase + i)) : (int)s_sp2[cbase + i]), cbase + i);
            if (n >= kmax) { lo = 0; hi = 0; }
        }
    }
    n_out = active ? n : 0;
}

// Phase 2: warp-cooperative continuation for one unsaturated event: the 32 lanes test 32 consecutive spiral
// cells at once; an exclusive scan over the lanes' accept counts restores the spiral order and the K cap.
template <bool STAGED, int THREADS>
__device__ __forceinline__ int bl_probe_coop(const dagr_geom_t &g, int64_t N, int p, const int2 me, int eb, int tidx0, int c_begin,
                                             int n, const uint32_t *s_pbin, const uint16_t *s_rng, const short *s_sp2,
                                             const int2 *s_ti, const int2 *__restrict__ ti, uint32_t *s_acc, int owner,
                                             int32_t *__restrict__ nbr, uint16_t *__restrict__ off)
{
    const int kmax = g.K - 1;
    const int lane = threadIdx.x & 31;
    for (int c0 = c_begin; c0 < g.ncell && n < kmax; c0 += 32) {
        const int c = c0 + lane;
        int cnt = 0, base = 0, hi = 0, acc = 0;
        if (c < g.ncell) {
            const int pix = tidx0 + s_sp2[c];
            const uint32_t rg = s_rng[pix * BL_NB + eb];
            hi = rg >> 8; cnt = hi - (int)(rg & 0xff);
            base = (int)(s_pbin[pix] >> 8);
            for (int k = 0; k < cnt; k++) {
                const int2 o = STAGED ? s_ti[base + hi - 1 - k] : __ldg(ti + base + hi - 1 - k);
                acc += (o.y < me.y && me.x - o.x <= g.dt_us) ? 1 : 0;
            }
        }
        int incl = acc;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
        const int tot = __shfl_sync(0xffffffffu, incl, 31);
        if (acc > 0) {
            int slot = n + incl - acc;
            for (int k = 0; k < cnt && slot < kmax; k++) {
                const int j = base + hi - 1 - k;
                const int2 o = STAGED ? s_ti[j] : __ldg(ti + j);
                if (o.y < me.y && me.x - o.x <= g.dt_us) {
                    if (STAGED) s_acc[slot * THREADS + owner] = ((uint32_t)j << 10) | (uint32_t)c;
                    else { nbr[(int64_t)slot * N + p] = j; off[(int64_t)slot * N + p] = (uint16_t)c; }
                    slot++;
                }
            }
        }
        n = min(n + tot, kmax);
    }
    return n;
}

// ---- conv_a phase 2 on tensor cores (TC instances, dagr_l1_build_tc) -----------------------------------------------------
// out = [32 nodes of a warp x 48] x [48 x 16]: k = 3u + ci for the 45 slot inputs A[u][ci], k = 45 + ci for the root inputs
// (polarity, x/W, y/H) of the node itself.  mma.sync.m16n8k8 TF32 in 3xTF32 form (common.cuh): 6 k-steps x 2 m-tiles x
// 2 n-tiles.  On CUDA cores the product is 768 FFMA per event, each with its weight from the constant bank.
// Every lane holds one node's row; the A fragments need other lanes' rows, which go through shared memory: per k-step the
// warp writes its 32 x 8 block and reads it back with two ldmatrix.x4 (one per m-tile).  The block lives in the warp's own
// columns of s_acc, rows 0..7: s_acc[q][tid] is read only by phase B of lane tid (and written by the probe of a lane of the
// same warp), so after the warp's __syncwarp those columns are dead until the next chunk's probe, which starts behind a CTA
// barrier.  No shared memory is added, so the lean instance keeps five CTAs per SM.
// Layout: 16-byte chunk h (k = 4h .. 4h+3) of node row r at s_acc row 4h + (r >> 3), byte 16 (r & 7) of the warp's 128-byte
// piece: each ldmatrix matrix (8 nodes, one chunk) is one 128-byte piece, the stores and loads are free of bank conflicts.
// The six k-steps are one chain of 18 mma per output through fresh (zeroed) fragments, about the length of one conv_b2 pass
// (15).  conv_b2 measured twice the largest oracle error when all its passes were chained (the tensor cores' fp32 accumulation
// truncates); splitting this chain in two groups summed with __fadd_rn needs 16 more registers, which spilled in all three
// instances.  An output depends only on its node's row and the fixed k order, so a node gets the same bits in every instance.
// Weight fragments: dagr_l1a_tc_weights, float4 [k-step 0..5][lane][n-tile] = (hi b0, hi b1, lo b0, lo b1).
#define BL_TC_KSTEPS 6
static_assert(8 * BL_TC_KSTEPS == 3 * DAGR_KU + 3 && BL_TC_KSTEPS * 32 * 2 * 4 == DAGR_L1A_TC_WFRAG_FLOATS, "48 = 45 slot + 3 root inputs");

// The lean instance runs phase B at its 72-register cap with the 45 accumulators live; phase 2 adds 16 C registers plus the
// fragments.  So the inputs k = 38 .. 44 are parked in rows 8..14 of the lane's own s_acc column (dead as well, see above)
// right after phase B and read back for k-steps 4 and 5.  ptxas still spills loop state around phase 2 (52 bytes stored,
// 92 loaded per thread and chunk; 5 CTAs per SM kept).
#define BL_TC_PARK0 38

// this lane's 8 inputs of k-step s (pk: the parked inputs, read back)
template <int s>
__device__ __forceinline__ void bl_tc_inputs(const float (&A)[DAGR_KU][3], const float pk[3 * DAGR_KU - BL_TC_PARK0], const float rt[3],
                                             float v[8])
{
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int k = 8 * s + j;
        v[j] = k < BL_TC_PARK0 ? A[k / 3][k % 3] : k < 3 * DAGR_KU ? pk[k - BL_TC_PARK0] : rt[k - 3 * DAGR_KU];
    }
}

// c (C fragments) += [warp's 32 rows x 8] x [8 x 16] for k-step s.  xw = shared address of the warp's s_acc columns.
// Warp-uniform.
template <int s, int THREADS>
__device__ __forceinline__ void bl_tc_kstep(const float v[8], uint32_t xw, const float4 *__restrict__ wfrag, float2 c[8])
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t row = xw + (lane >> 3) * (THREADS * 4) + 16 * (lane & 7);
    __syncwarp();                                                       // the previous k-step's block has been read
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" :: "r"(row), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" :: "r"(row + 4 * THREADS * 4), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7])
                 : "memory");
    __syncwarp();
    // matrix i = lane >> 3 of m-tile mt: nodes 16 mt + 8 (i & 1) + 0..7, chunk i >> 1
    const uint32_t la = xw + (4 * (lane >> 4) + ((lane >> 3) & 1)) * (THREADS * 4) + 16 * (lane & 7);
#pragma unroll
    for (int mt = 0; mt < 2; mt++) {
        uint32_t r[4], ah[4], al[4];
        ldsm_x4(la + 2 * mt * THREADS * 4, r);
#pragma unroll
        for (int i = 0; i < 4; i++) tf32_split(r[i], ah[i], al[i]);
#pragma unroll
        for (int nt = 0; nt < 2; nt++)
            mma_3xtf32(c[4 * mt + 2 * nt], c[4 * mt + 2 * nt + 1], ah, al, __ldg(wfrag + (s * 32 + lane) * 2 + nt));
    }
}

// work list: wl_hdr[0] = number of voxels beyond this instance's staging capacity (queued in wl_ids when `defer`, otherwise
// only counted and probed from global memory), wl_hdr[1] = pop cursor of the dense kernel
template <int CAP, int THREADS, bool TC>
__device__ __forceinline__ void bl_voxel(const dagr_geom_t &g, int64_t N, const int32_t *__restrict__ start, const int2 *__restrict__ ti,
                                         const uint32_t *__restrict__ xyb, const float *__restrict__ feat_s,
                                         const dagr_l1a_params_t &P, const float4 *__restrict__ wfrag, const int do_conv, const int min_idx,
                                         const int32_t *__restrict__ flags,
                                         int32_t *__restrict__ nbr, uint16_t *__restrict__ off, uint32_t *__restrict__ cellmask,
                                         float *__restrict__ xa, const int cell, unsigned char *smem_raw, BLTile &T, uint32_t &s_mask,
                                         int32_t *__restrict__ wl_hdr, int32_t *__restrict__ wl_ids, const int defer)
{
    const int per = g.ny1 * g.nx1;
    const int b = cell / per, rem = cell % per, cy = rem / g.nx1, cx = rem % g.nx1;
    const int p0 = start[(int64_t)cell * g.CP], p1 = start[(int64_t)(cell + 1) * g.CP];
    if (p1 == p0) { if (threadIdx.x == 0 && min_idx <= 0) cellmask[cell] = 0; return; }      // block-uniform

    // ---- shared memory carve-up -------------------------------------------------------------------
    const int TWmax = g.CW + 2 * g.r, THmax = g.CH + 2 * g.r, TPmax = TWmax * THmax, R = 2 * g.r + 1;
    // factor tables of the slot weights (tab[c][k+3j] == tabx[dx+r][k] * taby[dy+r][j]), laid out so that a warp's lookups
    // do not collide: wy[0..3] as one float4 per offset, wx as [3 x-slots][R] at a 4-byte stride, wy[4] apart
    float4 *s_wy = (float4 *)smem_raw;                                  // [R]
    float *s_wx = (float *)(s_wy + R);                                  // [3][R]
    float *s_wy4 = s_wx + 3 * R;                                        // [R]
    int2 *s_ti = (int2 *)(s_wy4 + R);                                   // [CAP]  (16-byte aligned: 32 R bytes of tables)
    float *s_feat = (float *)(s_ti + CAP);                              // [CAP]
    uint16_t *s_rng = (uint16_t *)(s_feat + CAP);                       // [TP][BL_NB]  lo | hi << 8   (16-byte aligned: CAP % 4 == 0)
    uint32_t *s_pbin = (uint32_t *)(s_rng + TPmax * BL_NB);             // [TP]  pos << 8 | visible count
    float *s_posx = (float *)(s_pbin + TPmax);                          // [TWmax]
    float *s_posy = s_posx + TWmax;                                     // [THmax]
    uint16_t *s_sp = (uint16_t *)(s_posy + THmax);                      // [ncell]  (dx + r) | (dy + r) << 5
    short *s_sp2 = (short *)(s_sp + g.ncell);                           // [ncell]  dy*TW + dx
    uint32_t *s_acc = (uint32_t *)(smem_raw + bl_acc_offset(g, CAP));   // [K-1][THREADS]  record << 10 | cell
    uint32_t *s_occ_r = s_acc + (DAGR_ELL - 1) * THREADS;               // [BL_NB][THmax] row occupancy bitmasks (ring walk)
    uint16_t *s_order = (uint16_t *)s_occ_r;                            // [THREADS]  (cell walk; see bl_smem_bytes)

    const int dtw = max(g.dt_us, 1);
    const float dtw_inv = 1.0f / (float)dtw;
    if (threadIdx.x == 0) {
        const int X0 = g.vx0[cx], X1 = g.vx0[cx + 1], Y0 = g.vy0[cy], Y1 = g.vy0[cy + 1];
        T.X0 = X0 - g.r; T.Y0 = Y0 - g.r; T.TW = X1 - X0 + 2 * g.r; T.TH = Y1 - Y0 + 2 * g.r;
        const int clo = max(cx - 1, 0), chi = min(cx + 1, g.nx1 - 1);
        int o = 0;
        for (int rr = 0; rr < 3; rr++) {
            const int ry = cy - 1 + rr;
            if (ry < 0 || ry >= g.ny1) { T.run_start[rr] = 0; T.run_len[rr] = 0; T.run_off[rr] = o; continue; }
            const int64_t c0 = (int64_t)b * per + ry * g.nx1 + clo, c1 = (int64_t)b * per + ry * g.nx1 + chi + 1;
            const int s = start[c0 * g.CP], e = start[c1 * g.CP];
            T.run_start[rr] = s; T.run_len[rr] = e - s; T.run_off[rr] = o;
            o += e - s;
        }
        T.smin = 0x7fffffff; T.smax = -0x7fffffff; T.unsorted = 0; T.maxidx = -1;
        s_mask = 0;
    }
    __syncthreads();
    const int TW = T.TW, TH = T.TH, TP = TW * TH;
    const bool use_rings = TW <= 32 && TH <= 32 && g.r <= 8;            // block-uniform (a ring = 8d <= 64 mask bits)
    uint32_t *s_occ_c = s_occ_r + BL_NB * TH;                           // [BL_NB][TW] column occupancy bitmasks
    const int total = T.run_off[2] + T.run_len[2];
    const bool staged = total <= CAP;                                   // block-uniform
    if (!staged && wl_hdr != nullptr) {
        // too many records for this instance's staging buffer: hand the voxel to the dense kernel (which runs next on
        // the stream) instead of probing global memory -- or, when the caller did not ask for that, just count it
        int slot = 0;
        if (threadIdx.x == 0) slot = atomicAdd(&wl_hdr[0], 1);
        if (defer) { if (threadIdx.x == 0) wl_ids[slot] = cell; return; }
    }
    const int bbase = b * per * g.CP;

    for (int i = threadIdx.x; i < g.ncell; i += blockDim.x) {
        const int dx = g.spiral[2 * i], dy = g.spiral[2 * i + 1];
        s_sp[i] = (uint16_t)((dx + g.r) | ((dy + g.r) << 5));
        s_sp2[i] = (short)(dy * TW + dx);
    }
    for (int i = threadIdx.x; i < R; i += blockDim.x) {
        const float4 tx = __ldg(reinterpret_cast<const float4 *>(g.tabx) + i);
        s_wx[i] = tx.x; s_wx[R + i] = tx.y; s_wx[2 * R + i] = tx.z;
        s_wy[i] = __ldg(reinterpret_cast<const float4 *>(g.taby) + 2 * i);
        s_wy4[i] = __ldg(g.taby + 8 * i + 4);
    }
    // ---- tile tables: per-pixel FIFO bin, normalised positions ----------------------------------------
    for (int i = threadIdx.x; i < TW; i += blockDim.x) {
        const int gx = T.X0 + i;
        s_posx[i] = (gx >= 0 && gx < g.W) ? g.posx0[gx] : 0.f;
    }
    for (int i = threadIdx.x; i < TH; i += blockDim.x) {
        const int gy = T.Y0 + i;
        s_posy[i] = (gy >= 0 && gy < g.H) ? g.posy0[gy] : 0.f;
    }
    for (int i = threadIdx.x; i < TP; i += blockDim.x) {
        const int ty = i / TW, tx = i % TW;
        const int gx = T.X0 + tx, gy = T.Y0 + ty;
        uint32_t v = 0;
        if (gx >= 0 && gx < g.W && gy >= 0 && gy < g.H) {
            const int ky = g.ykey[gy], kx = g.xkey[gx];
            const int k = bbase + ky + kx;
            const int s = start[k], e = start[k + 1];
            if (e > s) {
                const int lo = max(s, e - g.Q);                         // newest Q entries (ev_graph.cu:201-211)
                const int rr = ky / (g.nx1 * g.CP) - cy + 1;
                const int pos = staged ? (lo - T.run_start[rr] + T.run_off[rr]) : lo;
                v = ((uint32_t)pos << 8) | (uint32_t)(e - lo);
            }
        }
        s_pbin[i] = v;
    }
    // ---- stage the neighbourhood records (three coalesced runs) -------------------------------------
    if (staged) {
        for (int rr = 0; rr < 3; rr++) {
            const int s = T.run_start[rr], o = T.run_off[rr], len = T.run_len[rr];
            for (int i = threadIdx.x; i < len; i += blockDim.x) {
                s_ti[o + i] = ti[s + i];
                s_feat[o + i] = feat_s[s + i];
            }
        }
    }
    if (use_rings)
        for (int i = threadIdx.x; i < BL_NB * TW; i += blockDim.x) s_occ_c[i] = 0;
    // slice range of the voxel's own events
    {
        int mn = 0x7fffffff, mx = -0x7fffffff, mi = -1;
        for (int p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
            const int2 r = ti[p];
            if (r.y < min_idx) continue;                                // incremental mode: only new events are processed
            const int sl = bl_div(r.x, dtw, dtw_inv); mn = min(mn, sl); mx = max(mx, sl); mi = max(mi, r.y);
        }
        mn = __reduce_min_sync(0xffffffffu, mn); mx = __reduce_max_sync(0xffffffffu, mx); mi = __reduce_max_sync(0xffffffffu, mi);
        if ((threadIdx.x & 31) == 0) { atomicMin(&T.smin, mn); atomicMax(&T.smax, mx); atomicMax(&T.maxidx, mi); }
    }
    __syncthreads();
    if (T.maxidx < 0) return;                                           // block-uniform: no new event in this voxel
    // ---- per-pixel time-bucket ranges ---------------------------------------------------------------
    // bucket(t) = clamp(t/delta_t - (smin-1), 0, NB-1); an event in bucket e needs records of buckets {e-1, e}.
    const int sbase = T.smin - 1;
    bool bucketed = staged && (T.smax - sbase) < BL_NB && (flags == nullptr || flags[0] == 0);   // block-uniform
    // the ranges of tile pixel i -> s_rng[i]; returns bit e set when bucket e's range is non-empty
    auto pixel_ranges = [&](int i) -> uint32_t {
        const uint32_t pb = s_pbin[i];
        const int vis = pb & 0xff, base = pb >> 8;
        unsigned char cum[BL_NB + 1];
#pragma unroll
        for (int q = 0; q <= BL_NB; q++) cum[q] = 0;
        if (bucketed) {
            int prev = 0;
            for (int k = 0; k < vis; k++) {
                int bk = bl_div(s_ti[base + k].x, dtw, dtw_inv) - sbase;
                bk = min(max(bk, 0), BL_NB - 1);
                if (bk < prev) T.unsorted = 1;                          // benign race: any writer sets 1
                prev = bk;
#pragma unroll
                for (int q = 0; q <= BL_NB; q++) cum[q] += (bk < q) ? 1 : 0;
            }
        } else {
#pragma unroll
            for (int q = 1; q <= BL_NB; q++) cum[q] = (unsigned char)vis;
        }
        // the eight (lo | hi << 8) ranges of a pixel are one 16-byte store (eight 2-byte stores at a 16-byte lane stride
        // cost four wavefronts each)
        static_assert(BL_NB == 8, "one uint4 per pixel");
        uint32_t w[4], occ = 0;
#pragma unroll
        for (int e = 0; e < BL_NB; e += 2) {
            const uint32_t r0 = (uint32_t)cum[e > 0 ? e - 1 : 0] | ((uint32_t)cum[e + 1] << 8);
            const uint32_t r1 = (uint32_t)cum[e] | ((uint32_t)cum[e + 2] << 8);
            w[e >> 1] = r0 | (r1 << 16);
            occ |= (cum[e + 1] > cum[e > 0 ? e - 1 : 0] ? 1u : 0u) << e;
            occ |= (cum[e + 2] > cum[e] ? 1u : 0u) << (e + 1);
        }
        reinterpret_cast<uint4 *>(s_rng)[i] = make_uint4(w[0], w[1], w[2], w[3]);
        return occ;
    };
    for (int pass = 0; pass < 2; pass++) {
        if (use_rings) {
            // the occupancy bitmasks of the ring walk come out of the same pass: one warp per tile row (TW <= 32), lane = column.
            // A row word is one ballot per bucket; a lane ORs its column's bits over the warp's rows and adds them to the
            // (zeroed) column words with one atomicOr per bucket -- distinct words, so the atomics do not collide.
            const int lane = threadIdx.x & 31;
            uint32_t colm[BL_NB];
#pragma unroll
            for (int e = 0; e < BL_NB; e++) colm[e] = 0;
            for (int row = threadIdx.x >> 5; row < TH; row += blockDim.x >> 5) {      // warp-uniform
                const uint32_t occ = lane < TW ? pixel_ranges(row * TW + lane) : 0u;
#pragma unroll
                for (int e = 0; e < BL_NB; e++) {
                    const uint32_t m = __ballot_sync(0xffffffffu, (occ >> e) & 1u);
                    if (lane == e) s_occ_r[e * TH + row] = m;
                    colm[e] |= ((occ >> e) & 1u) << row;
                }
            }
            if (lane < TW) {
#pragma unroll
                for (int e = 0; e < BL_NB; e++)
                    if (colm[e]) atomicOr(&s_occ_c[e * TW + lane], colm[e]);
            }
        } else {
            for (int i = threadIdx.x; i < TP; i += blockDim.x) pixel_ranges(i);
        }
        __syncthreads();
        if (!bucketed || !T.unsorted) break;                            // block-uniform
        bucketed = false;                                               // records not time-sorted: redo without buckets
        if (use_rings) {
            for (int i = threadIdx.x; i < BL_NB * TW; i += blockDim.x) s_occ_c[i] = 0;
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) T.bucketed = bucketed;                        // read after the event loop's first barrier
    // ---- thread <-> event assignment in arrival order (time-homogeneous warps) ------------------------
    uint32_t mloc = 0;
    for (int pb = p0; pb < p1; pb += blockDim.x) {                      // chunk = own events [pb, pb + chunk)
        const int chunk = min((int)blockDim.x, p1 - pb);
        __syncthreads();
        // rank of each event of the chunk by arrival index (cell walk only: the ring walk does not need age-sorted warps)
        if (!use_rings && (int)threadIdx.x < chunk) {
            const int d = T.run_off[1] - T.run_start[1];               // staged position - sorted position (run 1)
            const int myidx = staged ? s_ti[d + pb + threadIdx.x].y : ti[pb + threadIdx.x].y;
            int rank = 0;
            for (int k = 0; k < chunk; k++) {
                const int oi = staged ? s_ti[d + pb + k].y : __ldg(&ti[pb + k].y);
                rank += (oi < myidx) ? 1 : 0;
            }
            s_order[rank] = (uint16_t)threadIdx.x;
        }
        __syncthreads();
        // arrival ranks are dealt round-robin to the warps: every warp gets the same share of the old
        // (unsaturated, slow) events of the voxel, so no warp is the straggler of the CTA
        const int nw = blockDim.x >> 5;
        // ring walk: warps of similar age leave the ring loop together -> contiguous arrival ranks per warp;
        // cell walk (fallback): ranks dealt round-robin so that no warp is the straggler
        const int rank = use_rings ? (int)threadIdx.x : (int)(threadIdx.x & 31) * nw + (int)(threadIdx.x >> 5);
        bool active = rank < chunk;
        const int p = pb + (active ? (use_rings ? rank : (int)s_order[rank]) : 0);
        int x = 0, y = 0;
        int2 me = make_int2(0, 0);
        if (active) {
            const uint32_t w = xyb[p];
            x = w & 0xfff; y = (w >> 12) & 0xfff;
            me = ti[p];
            active = me.y >= min_idx;
        }
        const int tx0 = active ? x - T.X0 : g.r, ty0 = active ? y - T.Y0 : g.r;
        int eb = 0;
        if (T.bucketed) eb = min(max(bl_div(me.x, dtw, dtw_inv) - sbase, 0), BL_NB - 1);
        int n;
        const int tidx0 = ty0 * TW + tx0;
        if (use_rings) {
            if (staged) bl_probe_rings<true, THREADS>(g, N, p, active, me, eb, tx0, ty0, TW, TH, s_pbin, s_rng, s_occ_r, s_occ_c, s_sp2, s_ti, ti, s_acc, nbr, off, n);
            else        bl_probe_rings<false, THREADS>(g, N, p, active, me, eb, tx0, ty0, TW, TH, s_pbin, s_rng, s_occ_r, s_occ_c, s_sp2, s_ti, ti, s_acc, nbr, off, n);
        } else {
            if (staged) bl_probe<true, THREADS>(g, N, p, active, me, eb, tidx0, BL_R1 < g.ncell ? BL_R1 : g.ncell, s_pbin, s_rng, s_sp2, s_ti, ti, s_acc, nbr, off, n);
            else        bl_probe<false, THREADS>(g, N, p, active, me, eb, tidx0, BL_R1 < g.ncell ? BL_R1 : g.ncell, s_pbin, s_rng, s_sp2, s_ti, ti, s_acc, nbr, off, n);
            // events still unsaturated after BL_R1 cells continue warp-cooperatively (32 cells per step), one at a time
            if (BL_R1 < g.ncell) {
                unsigned todo = __ballot_sync(0xffffffffu, active && n < g.K - 1);
                while (todo) {
                    const int src = __ffs(todo) - 1;
                    todo &= todo - 1;
                    const int ep = __shfl_sync(0xffffffffu, p, src);
                    const int2 eme = make_int2(__shfl_sync(0xffffffffu, me.x, src), __shfl_sync(0xffffffffu, me.y, src));
                    const int eeb = __shfl_sync(0xffffffffu, eb, src), etidx = __shfl_sync(0xffffffffu, tidx0, src);
                    const int en = __shfl_sync(0xffffffffu, n, src);
                    const int owner = (int)(threadIdx.x & ~31u) + src;
                    const int nn = staged ? bl_probe_coop<true, THREADS>(g, N, ep, eme, eeb, etidx, BL_R1, en, s_pbin, s_rng, s_sp2, s_ti, ti, s_acc, owner, nbr, off)
                                          : bl_probe_coop<false, THREADS>(g, N, ep, eme, eeb, etidx, BL_R1, en, s_pbin, s_rng, s_sp2, s_ti, ti, s_acc, owner, nbr, off);
                    if ((int)(threadIdx.x & 31) == src) n = nn;
                }
                __syncwarp();
            }
        }
        if (active) nbr[(int64_t)(DAGR_ELL - 1) * N + p] = n;
        // phase B: A_u = sum_e tab[c_e][u] * (polarity_src, x_src/W, y_src/H), converged over the ELL slots;
        // also translates the staged record index into the global sorted position and collects the voxel mask.
        // tab[c][k+3j] is rebuilt as wy[j] * wx[k] from the factor tables; __fmul_rn keeps the product from being contracted
        // into the FMA that consumes it, so every weight has the bits of the [ncell][16] table (geometry.py checks the identity).
        // A lane's table rows differ from its neighbours': one 64-byte global row per edge and lane touched ~28 L1 lines per
        // warp-wide load, the factors are conflict-free shared-memory loads.
        const float f0 = active ? feat_s[p] : 0.f, f1 = s_posx[tx0], f2 = s_posy[ty0];
        float A[DAGR_KU][3];
        {
            const int o = g.r;                                          // self loop: spiral cell 0, offset (0, 0)
            const float4 wya = s_wy[o];
            const float wy[5] = {wya.x, wya.y, wya.z, wya.w, s_wy4[o]}, wx[3] = {s_wx[o], s_wx[R + o], s_wx[2 * R + o]};
#pragma unroll
            for (int jy = 0; jy < 5; jy++)
#pragma unroll
                for (int k = 0; k < 3; k++) {
                    const float t = __fmul_rn(wy[jy], wx[k]);
                    A[k + 3 * jy][0] = t * f0; A[k + 3 * jy][1] = t * f1; A[k + 3 * jy][2] = t * f2;
                }
        }
        // tile position of spiral offset (-r, -r), x | y << 16: one register fewer through the loop (tile sides < 2^15)
        int txy = (tx0 - g.r) | ((ty0 - g.r) << 16);
        // the staged and the global-memory form are separate loops: one loop with both forms predicated needs more registers
        auto edges = [&](auto staged_c) {
            constexpr bool ST = decltype(staged_c)::value;
            for (int q = 0; q < n; q++) {
                const uint32_t e = (uint32_t)q * (uint32_t)N + (uint32_t)p;     // ELL index: 16 N < 2^28 (N < 2^24 checked)
                int j, c;
                if (ST) { const uint32_t a = s_acc[q * THREADS + threadIdx.x]; j = (int)(a >> 10); c = (int)(a & 0x3ff); }
                else { j = nbr[e]; c = off[e]; }
                const uint32_t sp = s_sp[c];
                const int dxi = (int)(sp & 31u), dyi = (int)(sp >> 5);
                const int txy_e = txy + dxi + (dyi << 16);
                const int tx = txy_e & 0xffff, ty = txy_e >> 16;
                // voxel row / column (0..2) of the source pixel: r is smaller than every voxel side (geometry.py), so the tile's
                // first and last r rows / columns belong to the neighbouring voxels and the rest to this one
                const int vr = (ty >= g.r) + (ty + g.r >= TH), vc = (tx >= g.r) + (tx + g.r >= TW);
                float e0;
                if (ST) {
                    e0 = s_feat[j];
                    nbr[e] = j - T.run_off[vr] + T.run_start[vr];
                    off[e] = (uint16_t)c;
                } else e0 = __ldg(feat_s + j);
                mloc |= 1u << (vr * 3 + vc);                            // bit 4 (this voxel) is dropped below
                const float e1 = s_posx[tx], e2 = s_posy[ty];
                const float4 wya = s_wy[dyi];
                const float wy[5] = {wya.x, wya.y, wya.z, wya.w, s_wy4[dyi]}, wx[3] = {s_wx[dxi], s_wx[R + dxi], s_wx[2 * R + dxi]};
#pragma unroll
                for (int jy = 0; jy < 5; jy++)
#pragma unroll
                    for (int k = 0; k < 3; k++) {
                        const int u = k + 3 * jy;
                        const float t = __fmul_rn(wy[jy], wx[k]);
                        A[u][0] = fmaf(t, e0, A[u][0]);
                        A[u][1] = fmaf(t, e1, A[u][1]);
                        A[u][2] = fmaf(t, e2, A[u][2]);
                    }
            }
        };
        if (staged) edges(std::true_type{});
        else        edges(std::false_type{});

        if constexpr (TC) {
            // the mma calls are warp-uniform: a lane without a node joins with its row (finite, and a row only reaches its
            // own outputs) and stores nothing
            if (!do_conv || !__any_sync(0xffffffffu, active)) continue;
            const uint32_t xw = bl_sa(s_acc) + 4u * (threadIdx.x & ~31u);
            float2 c[8];
#pragma unroll
            for (int i = 0; i < 8; i++) c[i] = make_float2(0.f, 0.f);
            constexpr int NPK = 3 * DAGR_KU - BL_TC_PARK0;
            const uint32_t own = bl_sa(s_acc) + 4u * threadIdx.x;
#pragma unroll
            for (int j = 0; j < NPK; j++) {
                const int k = BL_TC_PARK0 + j;
                bl_sts32(own + (8 + j) * THREADS * 4, __float_as_uint(A[k / 3][k % 3]));
            }
            float rt[3] = {0.f, 0.f, 0.f}, pk[NPK], v[8];
#pragma unroll
            for (int j = 0; j < NPK; j++) pk[j] = 0.f;
            bl_tc_inputs<0>(A, pk, rt, v); bl_tc_kstep<0, THREADS>(v, xw, wfrag, c);
            bl_tc_inputs<1>(A, pk, rt, v); bl_tc_kstep<1, THREADS>(v, xw, wfrag, c);
            bl_tc_inputs<2>(A, pk, rt, v); bl_tc_kstep<2, THREADS>(v, xw, wfrag, c);
            bl_tc_inputs<3>(A, pk, rt, v); bl_tc_kstep<3, THREADS>(v, xw, wfrag, c);
#pragma unroll
            for (int j = 0; j < NPK; j++) pk[j] = __uint_as_float(bl_lds32(own + (8 + j) * THREADS * 4));
            bl_tc_inputs<4>(A, pk, rt, v); bl_tc_kstep<4, THREADS>(v, xw, wfrag, c);
            // root inputs: read again rather than kept live through phase B (see the CUDA-core form below)
            int pr = p;
            asm volatile("" : "+r"(txy), "+r"(pr));
            rt[0] = __ldg(feat_s + pr); rt[1] = s_posx[(txy & 0xffff) + g.r]; rt[2] = s_posy[(txy >> 16) + g.r];
            bl_tc_inputs<5>(A, pk, rt, v); bl_tc_kstep<5, THREADS>(v, xw, wfrag, c);
            // BN + act straight from the C fragments: this lane holds channels 8 nt + 2t, +1 of nodes 16 mt + g and 16 mt + g + 8,
            // i.e. 8 bytes of the xa half-row nt (half-major [2][N][8], 16-byte chunks swizzled by XA_SWZ); the four lanes of a
            // row write its 32 bytes
            const int lane = threadIdx.x & 31, gq = lane >> 2, t = lane & 3;
            const int pv = active ? p : -1;
            float2 sc[2], sh[2];
#pragma unroll
            for (int nt = 0; nt < 2; nt++) {
                sc[nt] = *reinterpret_cast<const float2 *>(&P.scale[8 * nt + 2 * t]);
                sh[nt] = *reinterpret_cast<const float2 *>(&P.shift[8 * nt + 2 * t]);
            }
#pragma unroll
            for (int mt = 0; mt < 2; mt++)
#pragma unroll
                for (int hr = 0; hr < 2; hr++) {
                    const int q = __shfl_sync(0xffffffffu, pv, 16 * mt + 8 * hr + gq);
#pragma unroll
                    for (int nt = 0; nt < 2; nt++) {
                        const float2 o = c[4 * mt + 2 * nt + hr];
                        float r0 = fmaf(o.x, sc[nt].x, sh[nt].x), r1 = fmaf(o.y, sc[nt].y, sh[nt].y);
                        if (P.relu) { r0 = fmaxf(r0, 0.f); r1 = fmaxf(r1, 0.f); }
                        if (q >= 0)
                            *reinterpret_cast<float2 *>(xa + ((int64_t)nt * N + q) * 8 + (((t >> 1) ^ XA_SWZ(q)) << 2) + 2 * (t & 1)) =
                                make_float2(r0, r1);
                    }
                }
            continue;
        }
        if (!active || !do_conv) continue;
        // conv_a phase 2: out = sum_u W_u^T A_u + W_root^T x_i, BN, act  (weights in the constant bank)
        // the root term's inputs are read again rather than kept live through phase B, which keeps the lean instance within
        // its 72 registers; the empty asm hides that they are the values read before phase B, so the compiler neither reuses
        // those nor forms the addresses (and keeps them) before the loop
        int pr = p;
        asm volatile("" : "+r"(txy), "+r"(pr));
        const float r0 = __ldg(feat_s + pr), r1 = s_posx[(txy & 0xffff) + g.r], r2 = s_posy[(txy >> 16) + g.r];
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
            r = fmaf(r0, P.root[0][k], r);
            r = fmaf(r1, P.root[1][k], r);
            r = fmaf(r2, P.root[2][k], r);
            r = fmaf(r, P.scale[k], P.shift[k]);
            o[k] = P.relu ? fmaxf(r, 0.f) : r;
        }
        // xa is stored half-major [2][N][8] so that conv_b can stage one 32-byte channel half per pass
        const int sw = XA_SWZ(p);
        float4 *dst = reinterpret_cast<float4 *>(xa + (int64_t)p * 8);
        dst[sw] = make_float4(o[0], o[1], o[2], o[3]);
        dst[sw ^ 1] = make_float4(o[4], o[5], o[6], o[7]);
        dst = reinterpret_cast<float4 *>(xa + (N + (int64_t)p) * 8);
        dst[sw] = make_float4(o[8], o[9], o[10], o[11]);
        dst[sw ^ 1] = make_float4(o[12], o[13], o[14], o[15]);
    }
    mloc = __reduce_or_sync(0xffffffffu, mloc) & ~(1u << 4);
    if ((threadIdx.x & 31) == 0 && mloc) atomicOr(&s_mask, mloc);
    __syncthreads();
    if (threadIdx.x == 0) cellmask[cell] = (min_idx > 0 ? cellmask[cell] : 0u) | s_mask;
}



template <int CAP, int MIN_CTAS, bool TC>
__global__ void __launch_bounds__(BL_THREADS, MIN_CTAS)
k_l1_build(const dagr_geom_t g, int64_t N, const int32_t *__restrict__ start, const int2 *__restrict__ ti,
           const uint32_t *__restrict__ xyb, const float *__restrict__ feat_s,
           const __grid_constant__ dagr_l1a_params_t P, const float4 *__restrict__ wfrag, const int do_conv, const int min_idx,
           const int32_t *__restrict__ flags, int32_t *__restrict__ nbr, uint16_t *__restrict__ off, uint32_t *__restrict__ cellmask,
           float *__restrict__ xa, int32_t *__restrict__ wl_hdr, int32_t *__restrict__ wl_ids, const int defer)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ BLTile T;
    __shared__ uint32_t s_mask;
    bl_voxel<CAP, BL_THREADS, TC>(g, N, start, ti, xyb, feat_s, P, wfrag, do_conv, min_idx, flags, nbr, off, cellmask, xa,
                                  (int)blockIdx.x, smem_raw, T, s_mask, wl_hdr, wl_ids, defer);
}

// dense voxels: persistent CTAs (one per SM) pop voxel ids from the work list the regular kernel filled
template <bool TC>
__global__ void __launch_bounds__(BL_THREADS_BIG, 1)
k_l1_build_dense(const dagr_geom_t g, int64_t N, const int32_t *__restrict__ start, const int2 *__restrict__ ti,
                 const uint32_t *__restrict__ xyb, const float *__restrict__ feat_s,
                 const __grid_constant__ dagr_l1a_params_t P, const float4 *__restrict__ wfrag, const int do_conv, const int min_idx,
                 const int32_t *__restrict__ flags, int32_t *__restrict__ nbr, uint16_t *__restrict__ off,
                 uint32_t *__restrict__ cellmask, float *__restrict__ xa, int32_t *__restrict__ wl_hdr, const int32_t *__restrict__ wl_ids)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ BLTile T;
    __shared__ uint32_t s_mask;
    __shared__ int s_next;
    const int count = wl_hdr[0];
    for (;;) {
        __syncthreads();                                                // everyone is done with the previous voxel
        if (threadIdx.x == 0) s_next = atomicAdd(&wl_hdr[1], 1);
        __syncthreads();
        const int i = s_next;
        if (i >= count) break;
        bl_voxel<BL_CAP_BIG, BL_THREADS_BIG, TC>(g, N, start, ti, xyb, feat_s, P, wfrag, do_conv, min_idx, flags, nbr, off, cellmask, xa,
                                                 wl_ids[i], smem_raw, T, s_mask, nullptr, nullptr, 0);
    }
}

template <bool TC>
static int l1_build_launch(const dagr_geom_t *g, int64_t N, const int32_t *start, const int32_t *ti, const uint32_t *xyb,
                           const float *feat_s, const dagr_l1a_params_t *p_host, const float4 *wfrag, const int32_t *flags,
                           int min_idx, int32_t *nbr, uint16_t *off, uint32_t *cellmask, float *xa, int32_t *wl_hdr,
                           int32_t *wl_ids, int defer, cudaStream_t st)
{
    DAGR_CHECK_ARG(g, "null argument");
    static const dagr_l1a_params_t zero_params = {};
    const int do_conv = p_host != nullptr;
    if (!p_host) p_host = &zero_params;
    DAGR_CHECK_ARG(g->K >= 1 && g->K <= DAGR_ELL, "max_neighbors must be in [1,16]");
    DAGR_CHECK_ARG(g->r >= 0 && g->r <= 15 && g->Q <= 255, "radius must be <= 15 px and max_queue_size <= 255");
    DAGR_CHECK_ARG(N < (1ll << 24), "the staged probe packs positions in 24 bits (N < 16.7M per call)");
    const int cells = g->B * g->ny1 * g->nx1;
    const bool deferring = wl_hdr != nullptr && wl_ids != nullptr && defer;
    if (deferring) {
        const size_t smem = bl_smem_bytes(g, BL_CAP, BL_THREADS);
        auto kern = k_l1_build<BL_CAP, 4, TC>;
        DAGR_CUDA(dagr_allow_smem(kern, smem, true));
        kern<<<cells, BL_THREADS, smem, st>>>(*g, N, start, (const int2 *)ti, xyb, feat_s, *p_host, wfrag, do_conv, min_idx, flags, nbr,
                                              off, cellmask, xa, wl_hdr, wl_ids, 1);
    } else {
        const size_t smem = bl_smem_bytes(g, BL_CAP_LEAN, BL_THREADS);
        auto kern = k_l1_build<BL_CAP_LEAN, 5, TC>;
        DAGR_CUDA(dagr_allow_smem(kern, smem, true));
        kern<<<cells, BL_THREADS, smem, st>>>(*g, N, start, (const int2 *)ti, xyb, feat_s, *p_host, wfrag, do_conv, min_idx, flags, nbr,
                                              off, cellmask, xa, wl_hdr, wl_ids, 0);
    }
    DAGR_CHECK_LAUNCH();
    if (deferring) {
        const size_t smem_big = bl_smem_bytes(g, BL_CAP_BIG, BL_THREADS_BIG);
        static int n_sm = 0;
        if (n_sm == 0) {
            int dev = 0;
            DAGR_CUDA(cudaGetDevice(&dev));
            DAGR_CUDA(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        }
        auto kd = k_l1_build_dense<TC>;
        DAGR_CUDA(dagr_allow_smem(kd, smem_big));
        kd<<<n_sm, BL_THREADS_BIG, smem_big, st>>>(*g, N, start, (const int2 *)ti, xyb, feat_s, *p_host, wfrag, do_conv, min_idx, flags,
                                                   nbr, off, cellmask, xa, wl_hdr, wl_ids);
        DAGR_CHECK_LAUNCH();
    }
    return DAGR_OK;
}

extern "C" int dagr_l1_build(const dagr_geom_t *g, int64_t N, const int32_t *start, const int32_t *ti,
                             const uint32_t *xyb, const float *feat_s, const float *tab,
                             const dagr_l1a_params_t *p_host, const int32_t *flags, int min_idx, int32_t *nbr, uint16_t *off,
                             uint32_t *cellmask, float *xa, int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream)
{
    (void)tab;                                                          // the slot weights come from g->tabx / g->taby
    return l1_build_launch<false>(g, N, start, ti, xyb, feat_s, p_host, nullptr, flags, min_idx, nbr, off, cellmask, xa, wl_hdr,
                                  wl_ids, defer, (cudaStream_t)stream);
}

extern "C" int dagr_l1_build_tc(const dagr_geom_t *g, int64_t N, const int32_t *start, const int32_t *ti,
                                const uint32_t *xyb, const float *feat_s, const dagr_l1a_params_t *p_host, const float *wfrag,
                                const int32_t *flags, int min_idx, int32_t *nbr, uint16_t *off, uint32_t *cellmask, float *xa,
                                int32_t *wl_hdr, int32_t *wl_ids, int defer, void *stream)
{
    DAGR_CHECK_ARG(p_host && wfrag, "null params / weight fragments (dagr_l1a_tc_weights); the adjacency-only form is "
                                    "dagr_l1_build with p_host = NULL");
    return l1_build_launch<true>(g, N, start, ti, xyb, feat_s, p_host, (const float4 *)wfrag, flags, min_idx, nbr, off, cellmask, xa,
                                 wl_hdr, wl_ids, defer, (cudaStream_t)stream);
}

// host-side packing of the weight fragments of the TC instances (layout: see bl_tc_kstep): B[k][n] = w[k / 3][k % 3][n] for
// k < 45, root[k - 45][n] after that
extern "C" int dagr_l1a_tc_weights(const dagr_l1a_params_t *p_host, float *wfrag_host)
{
    DAGR_CHECK_ARG(p_host && wfrag_host, "null argument");
    auto B = [&](int k, int n) { return k < 3 * DAGR_KU ? p_host->w[k / 3][k % 3][n] : p_host->root[k - 3 * DAGR_KU][n]; };
    for (int s = 0; s < BL_TC_KSTEPS; s++)
        for (int lane = 0; lane < 32; lane++)
            for (int nt = 0; nt < 2; nt++) {
                const int gq = lane >> 2, t = lane & 3, n = 8 * nt + gq;
                const float x0 = B(8 * s + t, n), x1 = B(8 * s + t + 4, n);
                const float h0 = tf32_rna_host(x0), h1 = tf32_rna_host(x1);
                float *o = wfrag_host + (((size_t)s * 32 + lane) * 2 + nt) * 4;
                o[0] = h0; o[1] = h1; o[2] = x0 - h0; o[3] = x1 - h1;
            }
    return DAGR_OK;
}
