"""The event-level kernels' float64 reference, checked without a GPU.

tests/test_l1_kernels_gpu.py calls dagr_l1_build_tc / dagr_l1_build, dagr_l1_conv_b_pool_voxel_tc, dagr_l1_conv_a_image_tc /
_inc and dagr_xa_permute on synthetic event streams and compares them with the helpers below:
  * oracle_edges: the edges of oracle.ref_ops.RefGraph (graph_oracle.c) in arrival order -- per destination the self loop,
    then the neighbours in probe order.  The kernels' own nbr / off are never used by the reference; the GPU tests assert
    that they equal these edges mapped to sorted positions through the sort's perm;
  * ref_conv: oracle.ref_ops.spline_conv with (lut, remap) = build_lut(weight.double(), ...), called as
    oracle/ref_model.py calls it at the event level (Cartesian attribute of the fp32 normalised positions, clamped to
    [0, 1]).  The basis is the fp32 basis of that attribute (what the kernels evaluate, geometry.py checks that its table is
    an exact product of per-axis factors); weights, root, node features and every sum after it are float64.  The same call
    on |x|, |weight|, |root| gives S = sum |terms| of each output element's chain;
  * xa_pack / xa_unpack: the kernels' half-major node rows [2][N][8] with the 16-byte chunks of row p swapped where
    (p >> 2) & 1 (XA_SWZ), the inverse of Engine.xa_rows;
  * voxel_classes: the per-voxel instance selection of the kernels, restated from the sort's start table and the
    capacities the header publishes (DAGR_L1_*).

Error bound.  Every output element must satisfy |out - ref| <= c u S + 2 u |ref| (u = 2^-24), with c taken from the
operation counts of the kernel's chain (worst case, first order in u):
  * phase 1, A_u = sum over the n_e + 1 edges (self loop included) of tab * x: a chain of fp32 FMAs, one rounding each:
    (n_e + 1) u of sum |tab x|; through |W_u| into the output that is (n_e + 1) u S.  The slot weights tab = wy * wx are exact
    products (geometry.py), so they add nothing;
  * phase 2 in 3xTF32: A = hi + lo exactly (hi = cvt.rna.tf32(A)); the tensor cores read lo and the weights' lo at TF32
    precision (the low 13 bits are dropped: < 2^-10 |lo| <= 2^-21 |A| = 8 u |A| each), and lo * lo (<= 2^-22 = 4 u) is not
    formed: 20 u per product;
  * the tensor cores' fp32 accumulation truncates: 2 u per add, over the terms of one fragment chain -- 40 per conv pass
    (5 slots x 8 channels), 48 in the build kernel's single chain (45 slot inputs + 3 root inputs): 80 u and 96 u;
  * the convs add their 6 passes and 2 root k-steps into the result with __fadd_rn: 8 u;
  * epilogue: conv_b one BN FMA, the skip branch (3 FMAs + BN FMA, or skip_pre) and the add: 6 u; the image conv the
    add of the event-channel part and the BN FMA: 2 u, its skip output 19 FMAs + BN: 20 u; the build kernel BN: 2 u.
So C_BUILD_TC = 119, C_CONV = 115, C_IMAGE = 121 (the build kernel's part plus the image epilogue), C_SKIP = 20, plus n_e per element; the
fp32 dagr_l1_build's phase 2 is a chain of 48 x 3 FMAs without the split: C_BUILD_FP32 = 1 + 144 + 2 = 147.

Exact tier.  Geometries whose slot tables are dyadic and whose x / W, y / H are exact (512 x 512 at radius 6.5 / 512: den 32,
6 fractional bits; 1024 x 1024 at radius 14.5 / 1024: den 64, 8 bits), features and weights on coarse dyadic grids: every
phase-1 partial sum is an fp32 value, every A value splits exactly into two TF32 values, and every product and partial sum of
phase 2 and the epilogue is a multiple of one step g with |partial| <= S < 2^24 g.  Any summation order is then exact and the
kernels must equal float64 bit for bit.  exact_tier_budget() asserts this for given inputs.
"""
import contextlib
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
U = 2.0 ** -24
E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: the refused calls return before any CUDA call

C_BUILD_TC = 1 + 20 + 96 + 2
C_BUILD_FP32 = 1 + 144 + 2
C_CONV = 1 + 20 + 80 + 8 + 6
C_IMAGE = C_BUILD_TC + 2
C_SKIP = 20


def l1_caps():
    """the DAGR_L1_* staging capacities of include/dagr_b200.h"""
    text = (ROOT / "include" / "dagr_b200.h").read_text()
    return {k: int(v) for k, v in re.findall(r"#define DAGR_L1_([A-Z_]+)\s+(\d+)", text)}


# ------------------------------------------------------------------------------------------------------------------------
# node rows
# ------------------------------------------------------------------------------------------------------------------------
def _swz(N):
    return ((torch.arange(N) >> 2) & 1).bool()


def xa_pack(rows):
    """[N, 16] rows in sorted order -> the kernels' flat half-major [2 * N * 8] with XA_SWZ chunk swaps"""
    rows = rows.detach().cpu().float().clone()
    N = rows.shape[0]
    sw = _swz(N)
    rows[sw] = rows[sw].view(-1, 2, 2, 4).flip(2).reshape(-1, 16)
    return torch.cat([rows[:, :8].reshape(-1), rows[:, 8:].reshape(-1)])


def xa_unpack(flat, N):
    """inverse of xa_pack (the layout Engine.xa_rows reads)"""
    flat = flat.detach().cpu()
    rows = torch.cat([flat[:N * 8].view(N, 8), flat[N * 8:2 * N * 8].view(N, 8)], 1).clone()
    sw = _swz(N)
    rows[sw] = rows[sw].view(-1, 2, 2, 4).flip(2).reshape(-1, 16)
    return rows


# ------------------------------------------------------------------------------------------------------------------------
# events, graph, instance classes
# ------------------------------------------------------------------------------------------------------------------------
def make_events(W, H, B, n_bg, seed, clusters=(), border=0, empty=(), T=1_000_000):
    """batch i32[N], pos i32[N, 3] = (x, y, t) in arrival order: samples one after the other, time-sorted within each.
    n_bg uniform events per non-empty sample; clusters = (sample, x0, y0, w, h, n) boxes of n events; border events on the
    four sensor edges and in the last pool1 voxel column (x >= W - 4)."""
    rng = np.random.default_rng(seed)
    bs, xs, ys = [], [], []
    for b in range(B):
        if b in empty:
            continue
        x, y = [rng.integers(0, W, n_bg)], [rng.integers(0, H, n_bg)]
        for (cb, x0, y0, w, h, n) in clusters:
            if cb == b:
                x.append(rng.integers(x0, x0 + w, n)); y.append(rng.integers(y0, y0 + h, n))
        if border:
            k = border // 5
            x += [np.zeros(k, np.int64), np.full(k, W - 1), rng.integers(0, W, k), rng.integers(0, W, k), rng.integers(W - 4, W, k)]
            y += [rng.integers(0, H, k), rng.integers(0, H, k), np.zeros(k, np.int64), np.full(k, H - 1), rng.integers(0, H, k)]
        x, y = np.concatenate(x), np.concatenate(y)
        o = rng.permutation(len(x))
        bs.append(np.full(len(x), b)); xs.append(x[o]); ys.append(y[o])
    x, y, b = np.concatenate(xs), np.concatenate(ys), np.concatenate(bs)
    t = np.concatenate([np.sort(rng.integers(0, T, int((b == s).sum()))) for s in range(B) if s not in empty])
    return torch.from_numpy(b.astype(np.int32)), torch.from_numpy(np.stack([x, y, t], 1).astype(np.int32))


def oracle_edges(geom, batch, pos):
    """edge_index int64[2, E] = (src, dst) arrival ids from the graph oracle, in its order"""
    from oracle.ref_ops import RefGraph
    g = RefGraph(geom.W, geom.H, geom.B, geom.K, geom.Q, geom.r, geom.dt_us)
    return g.forward(batch, pos, delete_nodes=False, collect_edges=False)


def voxel_stats(geom, start):
    """(nown, total) int64[cells]: own nodes and nodes of the 3x3 voxel neighbourhood (clipped to the sample's grid)"""
    s = np.asarray(start, np.int64)
    nx, ny, B, CP = geom.nx1, geom.ny1, geom.B, geom.CP
    first = s[np.arange(B * ny * nx + 1) * CP]
    nown = first[1:] - first[:-1]
    total = np.zeros(B * ny * nx, np.int64)
    b, cy, cx = np.meshgrid(np.arange(B), np.arange(ny), np.arange(nx), indexing="ij")
    b, cy, cx = b.ravel(), cy.ravel(), cx.ravel()
    clo, chi = np.maximum(cx - 1, 0), np.minimum(cx + 1, nx - 1)
    for d in (-1, 0, 1):
        ry = cy + d
        ok = (ry >= 0) & (ry < ny)
        ryc = np.clip(ry, 0, ny - 1)
        row = (b * ny + ryc) * nx
        total += np.where(ok, first[row + chi + 1] - first[row + clo], 0)
    return nown, total


def voxel_classes(nown, total, caps):
    """boolean masks over the voxels: which instance each kernel runs on it (empty voxels are in no class)"""
    ne = nown > 0
    L, R, D = caps["BUILD_LEAN"], caps["BUILD"], caps["BUILD_DENSE"]
    c, cd = caps["CONV"], caps["CONV_DENSE"]
    sp = nown <= caps["SPARSE_NODES"]
    return {
        "build_lean_staged": ne & (total <= L), "build_lean_global": ne & (total > L),
        "build_staged": ne & (total <= R), "build_dense_staged": ne & (total > R) & (total <= D),
        "build_dense_global": ne & (total > D),
        "conv_staged": ne & (total <= c), "conv_dense_staged": ne & (total > c) & (total <= cd),
        "conv_dense_gathered": ne & (total > cd), "conv_gathered": ne & (total > c),
        "image_sparse_staged": ne & sp & (total <= c), "image_sparse_dense_staged": ne & sp & (total > c) & (total <= cd),
        "image_sparse_gathered": ne & sp & (total > c),
    }


def build_dense_smem_bytes(geom, cap=None, threads=512):
    """dynamic shared memory of dagr_l1_build's dense instance at this geometry, restated from build_l1.cu (bl_smem_bytes):
    factor tables, the staged records, the per-tile-pixel bins and time-bucket ranges, the spiral tables, the accepted-edge
    buffer and the ring-walk masks"""
    cap = l1_caps()["BUILD_DENSE"] if cap is None else cap
    TW, TH = geom.CW + 2 * geom.r, geom.CH + 2 * geom.r
    TP = TW * TH
    acc = (2 * geom.r + 1) * 32 + cap * 12 + TP * 4 + (TW + TH) * 4 + TP * 8 * 2 + geom.ncell * 4
    acc = (acc + 15) // 16 * 16
    return acc + 15 * threads * 4 + max(8 * (TW + TH) * 4, threads * 2) + 16


# ------------------------------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _chunk(elems):
    from oracle import ref_ops as R
    old = R.CHUNK_ELEMS
    R.CHUNK_ELEMS = elems
    try:
        yield
    finally:
        R.CHUNK_ELEMS = old


def slot_weights_25(geom, w15, seed=0):
    """[15, Cin, Cout] slot-major weights -> the [25, Cin, Cout] SplineConv weight; the unreachable spline kernels get
    arbitrary values (their basis weight is zero at every event-level offset)"""
    w15 = torch.as_tensor(w15).double()
    g = torch.Generator().manual_seed(seed)
    w25 = torch.randn((25,) + tuple(w15.shape[1:]), generator=g, dtype=torch.float64) * 100
    for u, s in enumerate(geom.slots1):
        w25[s] = w15[u]
    return w25


def ref_conv(geom, xin, edges, pos_xy, w15, root):
    """SplineConv at the event level in float64: xin [N, Cin] (arrival order), edges from oracle_edges, pos_xy int [N, 2]
    pixel positions, w15 [15, Cin, Cout] slot-major, root [Cin, Cout] -> (value, S) float64 [N, Cout]"""
    from oracle import ref_ops as R
    M = geom.effective_radius
    pos = torch.stack([geom.posx0[pos_xy[:, 0].long()], geom.posy0[pos_xy[:, 1].long()]], 1)      # fp32 x / W, y / H
    attr = torch.clamp(R.cartesian(pos, edges, M), min=0, max=1)
    w25 = slot_weights_25(geom, w15)
    root = torch.as_tensor(root).double()
    xin = torch.as_tensor(xin).double()
    out = []
    for f in (lambda t: t, torch.abs):
        lut, remap = R.build_lut(f(w25), geom.H, geom.W, geom.r, M, geom.r, M)
        with _chunk(4_000_000):
            out.append(R.spline_conv(f(xin), edges, attr, f(w25), f(root).t().contiguous(), lut=lut, remap=remap))
    return out[0], out[1]


def degrees(edges, N):
    """neighbours per node without the self loop (arrival order)"""
    dst = edges[1][edges[0] != edges[1]]
    return torch.bincount(dst, minlength=N)


def bound_ratio(out, ref, S, c):
    """max over elements of |out - ref| / (c u S + 2 u |ref|), c per element or scalar; NaN counts as infinite"""
    out, ref, S = torch.as_tensor(out).double(), torch.as_tensor(ref).double(), torch.as_tensor(S).double()
    err = (out - ref).abs()
    bound = torch.as_tensor(c, dtype=torch.float64) * U * S + 2 * U * ref.abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isnan(out), torch.full_like(err, float("inf")), r)
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------------------------------
# exact tier
# ------------------------------------------------------------------------------------------------------------------------
def dyadic(rng, shape, bits, exp):
    """integers in [-(2^bits - 1), 2^bits - 1] times 2^-exp"""
    return (rng.integers(-(2 ** bits - 1), 2 ** bits, shape) * 2.0 ** -exp).astype(np.float32)


def tf32_rna(x):
    """cvt.rna.tf32.f32 on finite values: round to nearest, ties away from zero, low 13 mantissa bits cleared"""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x1000) & 0xffffe000).astype(np.uint32).view(np.float32)


def splits_exactly(a):
    """every value is hi + lo with hi = rna_tf32(a) and lo a TF32 value (low 13 bits clear): the 3xTF32 product is exact"""
    a = np.asarray(a, np.float32)
    hi = tf32_rna(a)
    lo = (a - hi).astype(np.float32)
    return bool(np.all(hi.astype(np.float64) + lo == a.astype(np.float64)) and not (lo.view(np.uint32) & 0x1fff).any())


def grid_exact(v, step):
    """every value is a multiple of `step` below 2^24 step in magnitude: an exact fp32 value"""
    q = np.asarray(v, np.float64) / step
    return bool(np.all(q == np.round(q)) and np.all(np.abs(q) < 2.0 ** 24))


def exact_tier_budget(A_abs_max, a_step, S, g):
    """the exact-tier conditions: phase-1 values (|A| <= A_abs_max on the grid a_step) are fp32- and 3xTF32-exact (at most 21
    significant bits), and every phase-2 / epilogue partial sum (<= S on the grid g) is exact.  Returns the bits used."""
    a_bits = float(np.log2(max(A_abs_max, a_step) / a_step))
    s_bits = float(np.log2(max(float(np.max(S)), g) / g))
    if not (a_bits <= 21 and s_bits < 24):
        raise ValueError(f"inputs outside the exact tier: phase 1 needs {a_bits:.1f} bits, phase 2 {s_bits:.1f}")
    return a_bits, s_bits


# ------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------
def test_header_publishes_the_capacities_in_order():
    c = l1_caps()
    assert c["BUILD_LEAN"] <= c["BUILD"] < c["BUILD_DENSE"] and c["CONV"] < c["CONV_DENSE"], c
    assert c["SPARSE_NODES"] == 32, c
    src = (ROOT / "dagr_b200" / "csrc" / "build_l1.cu").read_text() + (ROOT / "dagr_b200" / "csrc" / "conv_l1.cu").read_text()
    assert not re.search(r"#define (BL|CB2)_CAP\w*\s+\d", src), "the capacities live in the header only"


@pytest.mark.parametrize("wh,radius,fits", [((640, 480), 0.01, True), ((1280, 720), 0.01, True), ((512, 512), 6.5 / 512, True),
                                            ((1280, 960), 0.01, False), ((1024, 1024), 14.5 / 1024, False)])
def test_dense_build_instance_fits_the_h100_only_below_large_voxels_at_large_radius(wh, radius, fits):
    """the H100's opt-in limit is 227 KB per block (232448 B); the GPU tests run both kinds of geometry with defer = 1"""
    from dagr_b200.geometry import Geometry
    geom = Geometry(*wh, 1, radius=radius, device="cpu")
    assert (build_dense_smem_bytes(geom) + 128 <= 232448) == fits, build_dense_smem_bytes(geom)


def test_xa_layout_round_trips_and_matches_the_engine_reader():
    from dagr_b200.engine import Engine
    N = 13
    rows = torch.arange(N * 16, dtype=torch.float32).view(N, 16)
    flat = xa_pack(rows)
    assert torch.equal(xa_unpack(flat, N), rows)
    # row 4 is swizzled: its first stored 16-byte chunk holds channels 4..7
    assert flat[4 * 8:4 * 8 + 4].tolist() == rows[4, 4:8].tolist() and flat[0:4].tolist() == rows[0, 0:4].tolist()

    class _E:
        last = dict(N=N, ws=dict(xa=flat))
    assert torch.equal(Engine.xa_rows(_E()), rows)


def test_bound_constants_follow_the_operation_counts():
    assert C_BUILD_TC == 119 and C_CONV == 115 and C_IMAGE == 121 and C_BUILD_FP32 == 147
    # one ulp-scale fault on a single term of a 16-edge chain of unit terms stays detectable: 16 edges x 16 channels of
    # unit terms give S = 256, the bound is (115 + 15) u S ~ 2^-9 -- a slot weight off by 2^-8 in one product is outside it
    S = 256.0
    assert (C_CONV + 15) * U * S < 2.0 ** -8


def test_exact_tier_budget_of_the_gpu_inputs_and_its_refusal():
    """512 x 512, r = 7: slot weights on 2^-6, x / W on 2^-9; build phase 1 sums n_e + 1 <= 16 edges of |e| <= 1: |A| <= 16
    on 2^-15 (20 bits), phase 2 with 3-bit weights on 2^-2.  conv_b: 4-bit features on 2^-2, |A| <= 16 * 3.75 on 2^-8"""
    from dagr_b200.geometry import Geometry
    geom = Geometry(512, 512, 1, radius=6.5 / 512, device="cpu")
    assert grid_exact(geom.tabx.numpy(), 2.0 ** -6) and grid_exact(geom.taby.numpy(), 2.0 ** -6)
    assert grid_exact(geom.posx0.numpy(), 2.0 ** -9) and grid_exact(geom.posy0.numpy(), 2.0 ** -9)
    geom2 = Geometry(1024, 1024, 1, radius=14.5 / 1024, device="cpu")
    assert geom2.r == 15 and geom2.den1_x == geom2.den1_y == 64.0
    assert grid_exact(geom2.tabx.numpy(), 2.0 ** -8) and grid_exact(geom2.taby.numpy(), 2.0 ** -8)
    # build: |A| <= 16, S <= 1.75 * (3 * 16 + 3)
    assert exact_tier_budget(16.0, 2.0 ** -15, np.array([1.75 * 51]), 2.0 ** -17)[1] < 24
    # conv_b: sum_u |A_u| <= 16 x 3.75 per channel, 16 channels + root, 3-bit weights; S <= 1.75 * 17 * 60
    assert exact_tier_budget(60.0, 2.0 ** -8, np.array([1.75 * 17 * 60]), 2.0 ** -10)[1] < 24
    # the 3xTF32 split of 20-bit A values is exact, of 24-bit values not
    rng = np.random.default_rng(0)
    a20 = (rng.integers(-(2 ** 20 - 1), 2 ** 20, 10000) * 2.0 ** -15).astype(np.float32)
    assert splits_exactly(a20)
    a24 = ((rng.integers(2 ** 22, 2 ** 23, 10000) * 2 + 1) * 2.0 ** -15).astype(np.float32)
    assert not splits_exactly(a24)
    with pytest.raises(ValueError, match="outside the exact tier"):
        exact_tier_budget(16.0, 2.0 ** -24, np.array([100.0]), 2.0 ** -17)          # x / W on 2^-18 (1024 x 1024 build)
    with pytest.raises(ValueError, match="outside the exact tier"):
        exact_tier_budget(16.0, 2.0 ** -15, np.array([1.75 * 51]), 2.0 ** -23)       # 9-bit weights


def test_voxel_classes_on_a_hand_built_start_table():
    """one sample, 3 x 2 voxels with CP = 1: totals clip at the grid's edges"""
    from types import SimpleNamespace
    geom = SimpleNamespace(nx1=3, ny1=2, B=1, CP=1)
    own = np.array([5, 0, 2000, 1, 1, 1])
    start = np.concatenate([[0], np.cumsum(own)])
    nown, total = voxel_stats(geom, start)
    assert nown.tolist() == own.tolist()
    assert total.tolist() == [5 + 0 + 1 + 1, 2008, 2002, 7, 2008, 2002]
    caps = dict(BUILD_LEAN=1536, BUILD=2048, BUILD_DENSE=12288, CONV=1344, CONV_DENSE=6144, SPARSE_NODES=32)
    k = voxel_classes(nown, total, caps)
    assert k["build_lean_global"].tolist() == [False, False, True, False, True, True]        # voxel 1 is empty
    assert k["conv_dense_staged"].sum() == 3 and k["image_sparse_dense_staged"].tolist() == [False] * 4 + [True, True]


def test_reference_conv_on_a_known_answer():
    """two events one pixel apart in x: node 1 reads node 0 at d = (-1, 0).  With all 25 kernels' weights = k (slot id) the
    message is sum_s basis_s * k_s * x: the basis of d / den + 0.5 for den = 32 (512 x 512, r = 7)"""
    from dagr_b200.geometry import Geometry
    geom = Geometry(512, 512, 1, radius=6.5 / 512, device="cpu")
    edges = torch.tensor([[0, 1, 0], [0, 1, 1]])
    pos = torch.tensor([[100, 50], [101, 50]])
    w15 = torch.zeros(15, 1, 1, dtype=torch.float64)
    c0 = [c for c, (dx, dy) in enumerate(geom.spiral.tolist()) if (dx, dy) == (-1, 0)][0]
    for u in range(15):
        w15[u] = float(u + 1)
    v, S = ref_conv(geom, torch.tensor([[2.0], [3.0]]), edges, pos, w15, torch.tensor([[0.5]]))
    tab = geom.tab1.double()
    self_msg = float((tab[0, :15] * torch.arange(1, 16)).sum())
    assert v[0, 0] == 2.0 * self_msg + 1.0
    assert v[1, 0] == 3.0 * self_msg + 2.0 * float((tab[c0, :15] * torch.arange(1, 16)).sum()) + 1.5
    assert torch.equal(S, v.abs())


# ---- argument contract ---------------------------------------------------------------------------------------------------
def _geom():
    from dagr_b200 import _lib
    g = _lib.Geom()
    g.W, g.H, g.B, g.T, g.r, g.K, g.nx1, g.ny1 = 640, 480, 1, 1000000, 7, 16, 56, 40
    return g


def _conv_b(lib, P, over):
    a = dict(g=C.byref(_geom()), N=10, start=BAD, xyb=BAD, ti=BAD, feat_s=BAD, xa=BAD, nbr=BAD, off=BAD, p=C.byref(P),
             wfrag=BAD, skip_pre=None, min_idx=0, persist=None, x1=None, cnt=BAD, pxy=BAD, tmean=BAD, tmax=BAD, xg=BAD,
             ldx=16, wl_hdr=None, wl_ids=None, defer=0, stream=None)
    a.update(over)
    return lib.dagr_l1_conv_b_pool_voxel_tc(*a.values())


CONV_B_NULLS = ["g", "start", "xyb", "ti", "feat_s", "xa", "nbr", "off", "p", "wfrag", "cnt", "pxy", "tmean", "tmax", "xg"]


@pytest.mark.parametrize("null", CONV_B_NULLS)
def test_conv_b_refuses_null_pointers(null):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _conv_b(lib, _lib.L1BParams(), {null: None}) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_l1_conv_b_pool_voxel_tc" in msg and "null" in msg, msg


@pytest.mark.parametrize("over,word", [(dict(N=-1), "N out of range"), (dict(N=1 << 31), "N out of range"),
                                       (dict(min_idx=-1), "min_idx"), (dict(ldx=15), "ldx"), (dict(ldx=0), "ldx"),
                                       (dict(min_idx=5), "persist"), (dict(min_idx=5, x1=BAD), "persist")])
def test_conv_b_refuses_bad_sizes_and_an_incremental_step_without_persist(over, word):
    """min_idx > 0 without persist would pool the new nodes alone (max) or divide their sum by all nodes (mean)"""
    from dagr_b200 import _lib
    lib = _lib.load()
    for pool_mean in (0, 1):
        P = _lib.L1BParams()
        P.pool_mean = pool_mean
        assert _conv_b(lib, P, over) == E_ARG, (over, pool_mean)
        msg = lib.dagr_last_error().decode()
        assert word in msg, msg


def _conv_a_image(lib, over):
    from dagr_b200 import _lib
    P = _lib.L1ImgParams()
    a = dict(g=C.byref(_geom()), N=10, start=BAD, xyb=BAD, feat_s=BAD, x0=BAD, nbr=BAD, off=BAD, p=C.byref(P), wfrag=BAD,
             xa=BAD, skipv=BAD, wl_hdr=None, wl_ids=None, defer=0, stream=None)
    a.update(over)
    return lib.dagr_l1_conv_a_image_tc(*a.values())


@pytest.mark.parametrize("null", ["g", "start", "xyb", "feat_s", "x0", "nbr", "off", "p", "wfrag", "xa", "skipv"])
def test_conv_a_image_refuses_null_pointers(null):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _conv_a_image(lib, {null: None}) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_l1_conv_a_image_tc" in msg and "null" in msg, msg


@pytest.mark.parametrize("N", [-1, 1 << 31])
def test_conv_a_image_refuses_n_out_of_range(N):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _conv_a_image(lib, dict(N=N)) == E_ARG
    assert "N out of range" in lib.dagr_last_error().decode()
