// capi.cu -- error plumbing, argument contract and workspace-size queries of the C-ABI (host only).
#include "common.cuh"
#include <stdarg.h>

static thread_local char g_err[512] = "";

void dagr_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char *dagr_last_error(void) { return g_err; }

// ---- raise-only opt-in shared memory (see common.cuh) ---------------------------------------------------------------
#include <map>
#include <mutex>
#include <utility>
cudaError_t dagr_allow_smem_impl(const void *kernel, size_t bytes, bool max_carveout)
{
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, size_t> allowed;          // (device, kernel) -> bytes granted so far
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(mu);
    auto it = allowed.find({dev, kernel});
    if (it != allowed.end() && it->second >= bytes) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) return e;
    if (max_carveout && it == allowed.end()) {
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
    }
    allowed[{dev, kernel}] = bytes;
    return cudaSuccess;
}
extern "C" int dagr_abi_version(void) { return DAGR_ABI_VERSION; }

#include <string.h>

extern "C" int64_t dagr_scan_blocks(int64_t n);

#define DAGR_UNSUPPORTED(cond, ...)                                            \
    do { if (cond) { dagr_set_error(__VA_ARGS__); return DAGR_E_UNSUPPORTED; } } while (0)

extern "C" int dagr_check_config(const dagr_geom_t *g, int64_t N, int cin0, int cout0, const char *activation)
{
    DAGR_CHECK_ARG(g != nullptr, "null geometry");
    DAGR_UNSUPPORTED(g->W < 1 || g->H < 1 || g->W > 4096 || g->H > 4096, "sensor size %dx%d: the packed (x, y, batch) word holds 12 bits "
                     "per coordinate (W, H <= 4096)", g->W, g->H);
    DAGR_UNSUPPORTED(g->B < 1 || g->B > 255, "batch size %d: the packed (x, y, batch) word holds 8 bits of sample index (B <= 255)", g->B);
    DAGR_UNSUPPORTED(g->K < 1 || g->K > DAGR_ELL, "max_neighbors %d: the ELL adjacency has %d slots per node (1 <= K <= %d)", g->K, DAGR_ELL, DAGR_ELL);
    DAGR_UNSUPPORTED(g->Q < 1 || g->Q > 255, "max_queue_size %d: per-pixel FIFO depths are kept in 8 bits (Q <= 255)", g->Q);
    DAGR_UNSUPPORTED(g->r < 0 || g->r > 15, "radius %d px: spiral offsets are packed in 5 bits per axis (r <= 15; the ring walk of the probe "
                     "covers r <= 8, larger radii take the cell walk)", g->r);
    DAGR_UNSUPPORTED(g->ncell != (2 * g->r + 1) * (2 * g->r + 1), "ncell %d != (2r+1)^2", g->ncell);
    DAGR_UNSUPPORTED(g->r >= g->CW || g->r >= g->CH, "radius %d px must be smaller than a pool1 voxel (%dx%d px): coarse edges would leave the "
                     "8-neighbourhood the voxel-grid layers assume", g->r, g->CW, g->CH);
    const int64_t nk = (int64_t)g->B * g->ny1 * g->nx1 * g->CP;
    DAGR_UNSUPPORTED(nk >= (1ll << 31), "B*ny1*nx1*CP = %lld sort keys: the graph sort's 32-bit sort key holds fewer than 2^31", (long long)nk);
    DAGR_UNSUPPORTED(g->NK != nk, "NK %d != B*ny1*nx1*CP = %lld", g->NK, (long long)nk);
    DAGR_UNSUPPORTED(N < 0 || N >= (1ll << 24), "N = %lld events per call: sorted positions are packed in 24 bits (N < 16.7 M)", (long long)N);
    DAGR_UNSUPPORTED(cout0 != 16 || (cin0 != 3 && cin0 != 19), "conv_block1 = Layer(%d -> %d): the event-level kernels implement 3 -> 16 (events "
                     "only) and 19 -> 16 (image fusion), i.e. base_width 0.5 as in every reference config", cin0, cout0);
    DAGR_UNSUPPORTED(activation != nullptr && strcmp(activation, "relu") != 0, "activation '%s': the fused epilogues implement relu (all reference "
                     "configs)", activation);
    return DAGR_OK;
}

extern "C" int dagr_event_workspace_bytes(const dagr_geom_t *g, int64_t N, dagr_event_ws_t *out)
{
    DAGR_CHECK_ARG(g != nullptr && out != nullptr && N >= 0, "bad argument");
    const int64_t n = N > 0 ? N : 1, nk = (int64_t)g->NK + 1, cells = (int64_t)g->B * g->ny1 * g->nx1;
    const int64_t nscan = nk > n + 1 ? nk : n + 1;                     // the exporter scans N + 1 degrees with the same scratch
    out->key = 4 * n; out->tmp = 4 * n;
    out->count = 4 * nk; out->start = 4 * nk;
    out->blocksums = 4 * (dagr_scan_blocks(nscan) + 2);
    out->perm = 4 * n; out->ti = 8 * n; out->xyb = 4 * n; out->feat_s = 4 * n;
    out->nbr = 4 * (int64_t)DAGR_ELL * n; out->off = 2 * (int64_t)DAGR_ELL * n;
    out->cellmask = 4 * cells;
    out->xa = 4 * 16 * n;
    out->wl_hdr = 8; out->wl_ids = 4 * cells;
    out->x1 = 4 * 16 * n;
    return DAGR_OK;
}

extern "C" int dagr_pool_workspace_bytes(int64_t parent_cells, int channels, dagr_pool_ws_t *out)
{
    DAGR_CHECK_ARG(out != nullptr && parent_cells > 0 && channels > 0, "bad argument");
    out->acc = parent_cells * channels * 8;                             // fp64 sums (mean) or ordered-int maxima: 8 bytes per entry
    out->possum = parent_cells * 3 * 8;
    out->ptmax = parent_cells * 4; out->pcnt = parent_cells * 4; out->pmask = parent_cells * 4;
    return DAGR_OK;
}
