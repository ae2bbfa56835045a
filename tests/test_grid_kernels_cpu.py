"""The pooled-grid kernels' float64 reference, checked without a GPU.

tests/test_grid_kernels_gpu.py calls dagr_grid_conv, dagr_grid_linear_bn, dagr_grid_pool / _finalize and dagr_head_finish
on synthetic voxel grids and compares them with the helpers below:
  * export_grid: the node and edge lists a grid stands for: valid cells, and for every set neighbour bit an edge
    src = dst + (dcx, dcy) when that cell is on the grid, in the same sample and valid.  It is the product's own
    dagr_b200/export.grid_edges, not an independent export; test_export_of_a_hand_built_grid pins it to an edge list
    written out by hand;
  * edge_attr: the fp32 pseudo-coordinate fl(fl(d / den) + 0.5) the kernels evaluate; its spline basis must be the one
    oracle.ref_ops.build_lut (init_lut) computes;
  * ref_grid_conv: oracle.ref_ops.spline_conv in float64 plus the epilogue (* scale + shift, + skip, relu); the same call
    on |x|, |W|, |root|, |bias| gives S_e = sum |terms| per output element (the spline basis is non-negative);
  * two tiers of input.  Exact: powers-of-two den, integer offsets and features / weights on a coarse dyadic grid, so that
    every partial sum of every output element is a multiple of one step g and |partial| <= S_e < 2^24 g: any summation
    order is then exact and the kernel must equal the reference bit for bit.  Realistic: random normal data, a real
    Geometry level's den, and the probabilistic bound |out - ref| <= 8 sqrt(n_e) u S_e + 2 u |ref| (u = 2^-24).
Also the argument contract of the two entry points that check their channel counts before any CUDA call.
"""
import contextlib
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

F32 = np.float32
U = 2.0 ** -24
LAMBDA = 8.0
E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: the calls below return before any CUDA call


# ------------------------------------------------------------------------------------------------------------------------
# grids, export, attributes
# ------------------------------------------------------------------------------------------------------------------------
def make_grid(rng, nx, ny, B, filled, p_valid=0.6, px_max=16, py_max=8):
    """cnt i32[cells], pxy i32[cells, 2], mask i32[cells] (all nine bits random, the centre bit too): samples in `filled`
    have p_valid of their cells valid, every other sample is empty.  Pixel positions are uniform in [0, px_max] x
    [0, py_max] on every cell (the kernels must ignore them on empty cells), so neighbour offsets span +-px_max / +-py_max."""
    per = nx * ny
    cnt = np.zeros(B * per, np.int32)
    for b in filled:
        cnt[b * per:(b + 1) * per] = (rng.random(per) < p_valid) * rng.integers(1, 9, per)
    pxy = np.stack([rng.integers(0, px_max + 1, B * per), rng.integers(0, py_max + 1, B * per)], 1).astype(np.int32)
    mask = rng.integers(0, 512, B * per).astype(np.int32)
    return cnt, pxy, mask


def export_grid(nx, ny, B, cnt, mask):
    """(valid cells int64[n], edge_index int64[2, E] over node ids = rank among the valid cells), via export.grid_edges"""
    from dagr_b200.export import grid_edges
    cnt, mask = torch.as_tensor(cnt), torch.as_tensor(mask)
    gs = SimpleNamespace(cnt=cnt, mask=mask, cells=B * ny * nx)
    return torch.nonzero(cnt > 0).flatten(), grid_edges(gs, SimpleNamespace(nx=nx, ny=ny))


def edge_attr(pxy, cells, edges, den_x, den_y):
    """fp32 [E, 2]: fl(fl(d / den) + 0.5) with d = pixel position of the source - that of the destination"""
    pxy = np.asarray(pxy)
    src, dst = cells[edges[0]].numpy(), cells[edges[1]].numpy()
    d = (pxy[src] - pxy[dst]).astype(F32)
    return np.stack([d[:, 0] / F32(den_x) + F32(0.5), d[:, 1] / F32(den_y) + F32(0.5)], 1).astype(F32)


# ------------------------------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _chunk(elems):
    """bound spline_conv's [E, Cin, Cout] float64 temporaries (the per-destination order does not change)"""
    from oracle import ref_ops as R
    old = R.CHUNK_ELEMS
    R.CHUNK_ELEMS = elems
    try:
        yield
    finally:
        R.CHUNK_ELEMS = old


def ref_grid_conv(g, x, weight, rootT, bias=None, scale=None, shift=None, skip=None, relu=False):
    """g: dict(nx, ny, B, cnt, pxy, mask, den_x, den_y); x: [cells, Cin] (the column block the kernel reads);
    weight [25, Cin, Cout], rootT [Cin, Cout], bias / scale / shift [Cout], skip [cells, Cout], any float type.
    -> (ref, S, n) float64 [cells, Cout]: the result, sum |terms| and the number of terms per element; empty cells 0."""
    from oracle import ref_ops as R
    cells, edges = export_grid(g["nx"], g["ny"], g["B"], g["cnt"], g["mask"])
    attr = torch.from_numpy(edge_attr(g["pxy"], cells, edges, g["den_x"], g["den_y"])).double()
    d = lambda t: None if t is None else torch.as_tensor(t).double()                   # noqa: E731
    x, weight, rootT, bias, scale, shift, skip = map(d, (x, weight, rootT, bias, scale, shift, skip))
    ncell, Cin, Cout = x.shape[0], weight.shape[1], weight.shape[2]

    def conv(f):
        with _chunk(4_000_000):
            v = R.spline_conv(f(x[cells]), edges, attr, f(weight), f(rootT).t().contiguous(),
                              None if bias is None else f(bias))
        if scale is not None:
            v = v * f(scale) + f(shift)
        if skip is not None:
            v = v + f(skip[cells])
        return v

    v, s = conv(lambda t: t), conv(torch.abs)
    if relu:
        v = v.clamp(min=0)
    deg = torch.bincount(edges[1], minlength=len(cells)).double()
    n = 4 * deg * Cin + Cin + 4
    ref, S, N = (torch.zeros((ncell, Cout), dtype=torch.float64) for _ in range(3))
    ref[cells], S[cells], N[cells] = v, s, n[:, None].expand(-1, Cout)
    return ref, S, N


def ref_linear_bn(cnt, x, wT, scale=None, shift=None):
    """float64 BN(x @ wT) on valid rows, 0 elsewhere -> (ref, S, n)"""
    x, wT = torch.as_tensor(x).double(), torch.as_tensor(wT).double()
    v, s = x @ wT, x.abs() @ wT.abs()
    if scale is not None:
        sc, sh = torch.as_tensor(scale).double(), torch.as_tensor(shift).double()
        v, s = v * sc + sh, s * sc.abs() + sh.abs()
    valid = torch.as_tensor(cnt)[:, None] > 0
    zero = torch.zeros_like(v)
    return torch.where(valid, v, zero), torch.where(valid, s, zero), torch.full_like(v, x.shape[1] + 2)


# ------------------------------------------------------------------------------------------------------------------------
# the two tiers
# ------------------------------------------------------------------------------------------------------------------------
def dyadic(rng, shape, bits, exp):
    """integers in [-(2^bits - 1), 2^bits - 1] times 2^-exp: at most `bits` significant bits, on the grid 2^-exp"""
    return (rng.integers(-(2 ** bits - 1), 2 ** bits, shape) * 2.0 ** -exp).astype(F32)


def check_exact_tier(S, step):
    """every partial sum is a multiple of `step` no larger than S_e: exact in fp32 (any order) iff S_e < 2^24 step"""
    worst = float((torch.as_tensor(S) / step).max())
    if not worst < 2.0 ** 24:
        raise ValueError(f"inputs outside the exact tier: max S_e / step = {worst:.4g} >= 2^24")
    return worst


def bound_ratio(out, ref, S, n):
    """max over elements of |out - ref| / (8 sqrt(n) u S + 2 u |ref|); an element with a zero bound must be exact"""
    out, ref = torch.as_tensor(out).double(), torch.as_tensor(ref).double()
    err = (out - ref).abs()
    bound = LAMBDA * torch.sqrt(n) * U * S + 2 * U * ref.abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isnan(out), torch.full_like(err, float("inf")), r)
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------
def test_export_of_a_hand_built_grid():
    """B = 2 samples of 3 x 2 cells.  Bits that point off the grid, at an empty cell, across the sample boundary (the
    bottom row of sample 0 pointing down) or at the centre (bit 4) give no edge; an empty destination gives none either."""
    nx, ny, B = 3, 2, 2
    bit = lambda dcx, dcy: 1 << ((dcy + 1) * 3 + (dcx + 1))                              # noqa: E731
    cnt = np.array([1, 1, 0,
                    2, 1, 1,
                    1, 0, 1,
                    1, 1, 1], np.int32)
    mask = np.zeros(12, np.int32)
    mask[0] = bit(1, 0) | bit(-1, 0) | bit(0, -1) | bit(1, 1) | bit(0, 0)       # -> 1, 4; off the grid twice; centre
    mask[1] = bit(1, 0) | bit(-1, 1)                                            # -> 2 is empty; -> 3
    mask[2] = bit(-1, 0)                                                        # empty destination
    mask[3] = bit(-1, 0) | bit(1, 0)                                            # off the left edge; -> 4
    mask[4] = bit(0, 1) | bit(1, 1) | bit(-1, -1) | bit(1, -1)                  # down: next sample; -> 0, 2 (empty)
    mask[5] = bit(-1, -1) | bit(-1, 0) | bit(1, 0)                              # -> 1, 4; right: cell 6 of sample 1
    mask[6] = bit(0, -1) | bit(-1, 0) | bit(0, 1)                               # up / left: sample 0; -> 9
    mask[9] = bit(0, -1) | bit(1, -1)                                           # -> 6, 7 (empty)
    mask[11] = bit(-1, 0) | bit(0, -1) | bit(-1, -1)                            # -> 10, 8, 7 (empty)
    cells, edges = export_grid(nx, ny, B, cnt, mask)
    assert cells.tolist() == [0, 1, 3, 4, 5, 6, 8, 9, 10, 11]
    node = {c: i for i, c in enumerate(cells.tolist())}
    want = sorted((node[s], node[d]) for s, d in [(1, 0), (4, 0), (3, 1), (4, 3), (0, 4), (1, 5), (4, 5), (9, 6),
                                                  (6, 9), (10, 11), (8, 11)])
    assert list(map(tuple, edges.t().tolist())) == want                         # (src, dst) order, like torch.unique


@pytest.mark.parametrize("wh", [(640, 480), (320, 215), (240, 180)])
def test_edge_attr_is_init_luts_for_real_den(wh):
    """the spline basis of fl(fl(d / den) + 0.5) with Geometry's den == the basis inside oracle.ref_ops.build_lut (init_lut,
    spline_conv.py:16-37) with the level's max_value, at every offset (dx, dy) a level produces and a few beyond, bit for
    bit, on all four levels.  A one-hot weight [25, 1, 25] turns the LUT into the basis of each offset over the 25 slots."""
    from dagr_b200.geometry import Geometry
    from oracle import ref_ops as R
    W, H = wh
    geom = Geometry(W, H, 1, device="cpu")
    onehot = torch.eye(25).view(25, 1, 25)
    for lv in geom.levels:
        M = lv.cart_max
        r = int(float(lv.den_x)) // 2 + 2                                       # |attr - 0.5| <= 0.5 and a little past it
        lut, _ = R.build_lut(onehot, H, W, r, M, r, M)
        d = torch.arange(-r, r + 1)
        cells = torch.arange(len(d))
        pxy = np.stack([d.numpy() + r, d.numpy() + r], 1)
        edges = torch.stack([cells, torch.full_like(cells, r)])                 # src = offset d, dst = the zero offset
        a = torch.from_numpy(edge_attr(pxy, cells, edges, lv.den_x, lv.den_y))
        ax, ay = a[:, 0].repeat_interleave(len(d)), a[:, 1].repeat(len(d))      # dx outer, dy inner, as build_lut's meshgrid
        basis, index = R.spline_basis(torch.stack([ax, ay], 1), 5, True, 1)
        mine = torch.zeros(len(ax), 25).scatter_add_(1, index, basis)
        assert torch.equal(mine, lut.reshape(-1, 25)), (W, H, float(lv.den_x), float(lv.den_y))


def test_exact_tier_check_rejects_wide_inputs():
    """the exact-tier inputs of the GPU tests pass the check with room; 16-bit weights on the same grid do not"""
    rng = np.random.default_rng(0)
    nx, ny, B, Cin, Cout = 9, 7, 2, 130, 8
    cnt, pxy, mask = make_grid(rng, nx, ny, B, [0, 1])
    g = dict(nx=nx, ny=ny, B=B, cnt=cnt, pxy=pxy, mask=mask, den_x=32.0, den_y=16.0)
    x = dyadic(rng, (nx * ny * B, Cin), 2, 2)
    for bits, ok in ((6, True), (16, False)):
        w, root = dyadic(rng, (25, Cin, Cout), bits, bits), dyadic(rng, (Cin, Cout), bits, bits)
        _, S, _ = ref_grid_conv(g, x, w, root)
        step = 2.0 ** -5 * 2.0 ** -2 * 2.0 ** -bits                      # basis (1/8 x 1/4) x feature x weight
        if ok:
            assert check_exact_tier(S, step) < 2.0 ** 23
        else:
            with pytest.raises(ValueError, match="outside the exact tier"):
                check_exact_tier(S, step)


def test_reference_conv_on_a_known_answer():
    """one edge at attr (0.125, 0.5) (spline_kats.json: basis 0.5 / 0.5 at slots 10 / 11) into a cell with root term"""
    nx, ny, B = 2, 1, 1
    cnt, mask = np.array([1, 1], np.int32), np.array([0, 1 << 3], np.int32)            # cell 1 reads cell 0 (dcx = -1)
    pxy = np.array([[0, 0], [24, 0]], np.int32)                                           # d = (-24, 0): -24 / 64 + 0.5
    g = dict(nx=nx, ny=ny, B=B, cnt=cnt, pxy=pxy, mask=mask, den_x=64.0, den_y=16.0)
    w = torch.zeros(25, 1, 1, dtype=torch.float64)
    w[10], w[11], w[15], w[16] = 3.0, 5.0, -100.0, -100.0                     # 15 / 16 carry zero basis weight
    args = (g, np.array([[2.0], [7.0]]), w, torch.tensor([[0.5]]))
    kw = dict(bias=torch.tensor([1.0]), scale=torch.tensor([-2.0]), shift=torch.tensor([0.25]),
              skip=torch.tensor([[0.0], [-0.5]]))
    ref, S, n = ref_grid_conv(*args, **kw)
    v = (0.5 * 2 * 3 + 0.5 * 2 * 5 + 7 * 0.5 + 1.0) * -2.0 + 0.25 - 0.5
    assert ref[:, 0].tolist() == [(2 * 0.5 + 1.0) * -2.0 + 0.25, v]
    assert S[1, 0] == (0.5 * 2 * 3 + 0.5 * 2 * 5 + 7 * 0.5 + 1.0) * 2.0 + 0.25 + 0.5 and n[1, 0] == 4 + 1 + 4
    assert ref_grid_conv(*args, **kw, relu=True)[0][:, 0].tolist() == [0.0, 0.0]


def _grid_conv(lib, gr, Cin=16, Cout=16, ldin=0):
    return lib.dagr_grid_conv(gr, BAD, BAD, BAD, BAD, ldin, Cin, Cout, BAD, BAD, None, None, None, None, 0, 32.0, 16.0,
                              BAD, None)


@pytest.mark.parametrize("kw", [dict(Cin=0), dict(Cin=-5), dict(Cout=0), dict(Cout=-1), dict(Cin=16, ldin=15),
                                dict(Cin=130, ldin=1)])
def test_grid_conv_rejects_bad_channels(kw):
    from dagr_b200 import _lib
    lib = _lib.load()
    gr = _lib.Grid(nx=7, ny=5, B=1, W=640, H=480, posxr=None, posyr=None)
    assert _grid_conv(lib, gr, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_grid_conv" in msg and "bad channels" in msg, msg


@pytest.mark.parametrize("Cin,Cout", [(1537, 64), (4096, 8), (0, 64), (64, 0)])
def test_grid_linear_bn_rejects_bad_channels(Cin, Cout):
    """8 rows of Cin floats must fit the kernel's 48 KB of shared memory (Cin <= 1536)"""
    from dagr_b200 import _lib
    lib = _lib.load()
    assert lib.dagr_grid_linear_bn(100, BAD, BAD, Cin, Cout, BAD, BAD, BAD, BAD, None) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_grid_linear_bn" in msg and "bad channels" in msg, msg
