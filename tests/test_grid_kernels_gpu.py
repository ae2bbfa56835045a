"""The pooled-grid kernels of coarse.cu on their own, on synthetic voxel grids, through the C-ABI.

dagr_grid_conv against oracle.ref_ops.spline_conv in float64 (tests/test_grid_kernels_cpu.py) at every shipped
(Cin, Cout) and in each of its four kernels -- k_grid_conv_sk<16>, <4>, <1> and the one-warp-per-voxel k_grid_conv --
chosen by sizing the grid against the SM count; the kernel that ran is reported by the library
(dagr_grid_conv_last_instance), so the coverage cannot silently move.  (torch.profiler traces on the H100 drop a kernel's
record now and then, several sessions in a row, so they cannot carry an assertion that must never flake.)  Each case runs two tiers: exact inputs (dyadic, every partial sum exact: torch.equal) and realistic ones
(random normal, a real level's den, folded BN: per element |out - ref| <= 8 sqrt(n_e) u S_e + 2 u |ref|).  Grids have a
partial last CTA, empty samples and empty cells (output prefilled with NaN: every element must be written), and mask bits
that point off the grid, at empty cells, across a sample boundary and at the centre.  Then dagr_grid_linear_bn against a
float64 matmul, dagr_grid_pool / _finalize against float64 group max / mean bit for bit (and its error flag),
dagr_head_finish against torch fp32 and an ulp bound from CUDA's documented expf error, and a sample's rows of every
coarse kernel at B in {1, 2, 17, 31, 127} against its B = 1 run, bit for bit.
"""
from functools import lru_cache

import numpy as np
import pytest
import torch

from tests.test_grid_kernels_cpu import (U, bound_ratio, check_exact_tier, dyadic, edge_attr, export_grid, make_grid,
                                         ref_grid_conv, ref_linear_bn)

pytestmark = pytest.mark.gpu

NX, NY = 13, 7                          # 91 cells per sample: odd, so batches leave partial CTAs of 16 and 4
INSTANCES = ("sk16", "sk4", "sk1", "v1")


def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def instance(Cin, Cout, cells, nsm):
    """the kernel dagr_grid_conv picks (coarse.cu: CTAs to fill every SM, then shared memory per instance)"""
    per_cell = (26 * Cin + (0 if Cout <= 64 else 8 * Cout)) * 4

    def fits(cpb):
        a, p = 26 * Cin * cpb * 4, 8 * cpb * Cout * 4
        return (max(a, p) if Cout <= 64 else a + p) <= 200 * 1024
    if cells >= nsm * 32 and per_cell * 16 <= 110 * 1024 and fits(16):
        return "sk16"
    if cells >= nsm * 4 and per_cell * 4 <= 160 * 1024 and fits(4):
        return "sk4"
    return "sk1" if fits(1) else "v1"


def batch_for(size, nsm, per=NX * NY):
    """B with B * per cells in the size class ("big" >= 32 n_sm, "mid" in [4, 32) n_sm, "small" < 4 n_sm), not a multiple
    of 16 cells"""
    B = {"big": -(-32 * nsm // per) + 1, "mid": -(-4 * nsm // per) + 1, "small": max(2, (4 * nsm - 1) // per - 1)}[size]
    return B + 1 if (B * per) % 16 == 0 else B


LAST_INSTANCE = {16: "sk16", 4: "sk4", 1: "sk1", 0: "v1"}


def dev(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a) if isinstance(a, np.ndarray) else a)
    return (t if dtype is None else t.to(dtype)).cuda()


def grid(nx, ny, B, W=640, H=480, posxr=None, posyr=None):
    from dagr_b200 import _lib
    return _lib.Grid(nx=nx, ny=ny, B=B, W=W, H=H, posxr=None if posxr is None else posxr.data_ptr(),
                     posyr=None if posyr is None else posyr.data_ptr())


def run_grid_conv(g, xfull, off, ldin, Cin, Cout, p):
    """launch dagr_grid_conv on the column block xfull[:, off:off + Cin] -> (out fp32 [cells, Cout] on the host, instances)"""
    from dagr_b200 import _lib
    lib = _lib.load()
    cells = g["B"] * g["ny"] * g["nx"]
    d = {k: None if p.get(k) is None else dev(p[k], torch.float32) for k in ("w", "root", "bias", "scale", "shift", "skip")}
    cnt, pxy, mask, x = dev(g["cnt"]), dev(g["pxy"]), dev(g["mask"]), dev(xfull, torch.float32)
    out = torch.full((cells, Cout), float("nan"), device="cuda")
    _lib.check(lib.dagr_grid_conv(grid(g["nx"], g["ny"], g["B"]), _lib.ptr(cnt), _lib.ptr(pxy), _lib.ptr(mask),
                                  _lib.ptr(x[:, off:]), ldin, Cin, Cout, _lib.ptr(d["w"]), _lib.ptr(d["root"]),
                                  _lib.ptr(d["bias"]), _lib.ptr(d["scale"]), _lib.ptr(d["shift"]), _lib.ptr(d["skip"]),
                                  1 if p.get("relu") else 0, g["den_x"], g["den_y"], _lib.ptr(out), _lib.stream_ptr()),
               "dagr_grid_conv")
    torch.cuda.synchronize()
    return out.cpu(), {LAST_INSTANCE[lib.dagr_grid_conv_last_instance()]}


@lru_cache(None)
def real_den():
    """den of the convs after pool2 at 320 x 215 (64, 43: the y offsets are not dyadic)"""
    from dagr_b200.geometry import Geometry
    lv = Geometry(320, 215, 1, device="cpu").levels[1]
    return lv.den_x, lv.den_y


def conv_params(rng, tier, cells, Cin, Cout, flags):
    """weights and epilogue of one tier; flags: subset of 'bias', 'scale', 'skip', 'relu' -> (params, exact step)"""
    if tier == "exact":
        p = dict(w=dyadic(rng, (25, Cin, Cout), 6, 6), root=dyadic(rng, (Cin, Cout), 6, 6), bias=dyadic(rng, Cout, 6, 6),
                 scale=dyadic(rng, Cout, 2, 1), shift=dyadic(rng, Cout, 6, 6),
                 skip=dyadic(rng, (cells, Cout), 6, 6) if "skip" in flags else None)
    else:
        gamma, beta = rng.uniform(0.5, 1.5, Cout), rng.normal(0, 0.2, Cout)
        mean, var = rng.normal(0, 0.3, Cout), rng.uniform(0.3, 2.0, Cout)
        scale = (gamma / np.sqrt(var + 1e-5)).astype(np.float32)
        p = dict(w=(rng.standard_normal((25, Cin, Cout)) / np.sqrt(4 * Cin)).astype(np.float32),
                 root=(rng.standard_normal((Cin, Cout)) / np.sqrt(Cin)).astype(np.float32),
                 bias=rng.normal(0, 0.1, Cout).astype(np.float32), scale=scale,
                 shift=(beta - mean * scale).astype(np.float32),
                 skip=rng.standard_normal((cells, Cout)).astype(np.float32) if "skip" in flags else None)
    for k in ("bias", "scale", "skip"):
        if k not in flags:
            p[k] = None
    if p["scale"] is None:
        p["shift"] = None
    p["relu"] = "relu" in flags
    return p, 2.0 ** -13 * (0.5 if p["scale"] is not None else 1.0)


def conv_case(Cin, Cout, size, block=False, flags=("bias", "scale", "skip"), seed=0, off=0, ldin=0):
    """run both tiers of one grid-conv case; asserts; returns {tier: (instance, error / bound ratio or 0)}.  The kernel
    reads columns [off, off + Cin) of a [cells, ldin] array whose other columns are NaN (ldin = 0: a dense [cells, Cin]
    input); block = True is the second half of [cells, 2 Cin]."""
    if block:
        off, ldin = Cin, 2 * Cin
    nsm = n_sm()
    B = 4 if size == "v1" else batch_for(size, nsm)
    cells = B * NX * NY
    want = instance(Cin, Cout, cells, nsm)
    res = {}
    for tier in ("exact", "realistic"):
        rng = np.random.default_rng([seed, Cin, Cout, B, tier == "exact"])
        filled = [0, B - 1] if Cout > 1000 else sorted({0, 1, B // 2, B - 2, B - 1})
        den = (32.0, 16.0) if tier == "exact" else real_den()
        cnt, pxy, mask = make_grid(rng, NX, NY, B, filled, px_max=int(den[0]) // 2, py_max=int(den[1]) // 2)
        if tier == "exact":                       # many x offsets of +-16 (attr 0 and 1.0) and 0 (attr 0.5, a slot edge)
            pxy[0::3, 0], pxy[1::3, 0] = 0, 16
        g = dict(nx=NX, ny=NY, B=B, cnt=cnt, pxy=pxy, mask=mask, den_x=den[0], den_y=den[1])
        x = dyadic(rng, (cells, Cin), 2, 2) if tier == "exact" else rng.standard_normal((cells, Cin)).astype(np.float32)
        p, step = conv_params(rng, tier, cells, Cin, Cout, flags)
        xfull = x
        if ldin:                                  # a column block of a wider array; the other columns are NaN
            xfull = np.full((cells, ldin), np.nan, np.float32)
            xfull[:, off:off + Cin] = x
        out, seen = run_grid_conv(g, xfull, off, ldin, Cin, Cout, p)
        assert seen == {want}, f"{Cin}x{Cout} on {cells} cells: ran {seen}, expected {want}"
        ref, S, n = ref_grid_conv(g, x, p["w"], p["root"], p["bias"], p["scale"], p["shift"], p["skip"], p["relu"])
        what = f"{Cin}x{Cout} {want} {tier} (B = {B}, columns {off}.. of {ldin or Cin}, flags {'/'.join(flags) or '-'})"
        if tier == "exact":
            cells_v, edges = export_grid(NX, NY, B, cnt, mask)
            a = edge_attr(pxy, cells_v, edges, *den)
            assert {0.0, 1.0} <= set(a[:, 0].tolist()) and (a * 4 == np.floor(a * 4)).all(1).any(), what
            check_exact_tier(S, step)
            bad = (out.double() != ref).nonzero()
            assert len(bad) == 0, (f"{what}: {len(bad)} elements differ, first [cell, o] {bad[0].tolist()}: "
                                   f"{out[tuple(bad[0])].item()!r} != {ref[tuple(bad[0])].item()!r}")
            res[tier] = (want, 0.0)
        else:
            r = bound_ratio(out, ref, S, n)
            print(f"{what}: max |err| / bound = {r:.3g}")
            assert r <= 1.0, f"{what}: error {r:.3g} x the bound"
            res[tier] = (want, r)
    return res


# (Cin, Cout, column block): a few layer / head convs, 18 -> 128 (<16> with a separate partial-sum buffer) and 16 -> 6400
# (too wide for every split-K instance: k_grid_conv).  Every shape the shipped configurations launch, derived from the
# models, runs in tests/test_coarse_shapes_gpu.py.
SHAPES = [(18, 64, False), (66, 64, False), (64, 64, False), (66, 128, False), (130, 128, False), (128, 256, False),
          (96, 192, False), (32, 100, True), (64, 5, True)]
CASES = ([(ci, co, blk, "big") for ci, co, blk in SHAPES if instance(ci, co, 10 ** 6, 132) == "sk16"]
         + [(18, 128, False, "big")]
         + [(ci, co, blk, s) for ci, co, blk in SHAPES for s in ("mid", "small")]
         + [(16, 6400, False, "v1")])


def test_grid_conv_cases_reach_every_instance():
    nsm = n_sm()
    got = {instance(ci, co, (4 if s == "v1" else batch_for(s, nsm)) * NX * NY, nsm) for ci, co, _, s in CASES}
    assert got == set(INSTANCES), got


@pytest.mark.parametrize("Cin,Cout,block,size", CASES, ids=[f"{c[0]}x{c[1]}-{c[3]}" for c in CASES])
def test_grid_conv_vs_float64(Cin, Cout, block, size):
    conv_case(Cin, Cout, size, block)


@pytest.mark.parametrize("mask", range(16))
def test_grid_conv_epilogue_combinations(mask):
    """every combination of bias / scale (with shift) / skip / relu at 66 -> 64"""
    flags = tuple(f for i, f in enumerate(("bias", "scale", "skip", "relu")) if (mask >> i) & 1)
    conv_case(66, 64, "mid", flags=flags, seed=100 + mask)


# ------------------------------------------------------------------------------------------------------------------------
# linear + BN
# ------------------------------------------------------------------------------------------------------------------------
def run_linear_bn(cnt, x, wT, scale, shift):
    from dagr_b200 import _lib
    lib = _lib.load()
    cells, Cin = x.shape
    Cout = wT.shape[1]
    d_cnt, d_x, d_w = dev(cnt), dev(x), dev(wT)
    d_sc, d_sh = (None, None) if scale is None else (dev(scale), dev(shift))
    out = torch.full((cells, Cout), float("nan"), device="cuda")
    _lib.check(lib.dagr_grid_linear_bn(cells, _lib.ptr(d_cnt), _lib.ptr(d_x), Cin, Cout, _lib.ptr(d_w), _lib.ptr(d_sc),
                                       _lib.ptr(d_sh), _lib.ptr(out), _lib.stream_ptr()), "dagr_grid_linear_bn")
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("Cin,Cout,cells,bn", [(66, 64, 1003, True), (18, 128, 77, True), (130, 256, 515, False),
                                               (7, 130, 13, True), (96, 192, 9, False), (1536, 3, 21, True)])
def test_grid_linear_bn_vs_float64(Cin, Cout, cells, bn):
    """Cin not a multiple of 8 (clamped rows), cells not a multiple of 8, Cout above 128, scale = NULL"""
    linear_bn_case(Cin, Cout, cells, bn)


def linear_bn_case(Cin, Cout, cells, bn):
    """both tiers of dagr_grid_linear_bn on `cells` rows, 70 % of them valid, against the float64 matmul"""
    rng = np.random.default_rng([Cin, Cout, cells])
    cnt = (rng.random(cells) < 0.7).astype(np.int32)
    for tier in ("exact", "realistic"):
        if tier == "exact":
            x, wT = dyadic(rng, (cells, Cin), 3, 3), dyadic(rng, (Cin, Cout), 8, 8)
            scale, shift = (dyadic(rng, Cout, 2, 1), dyadic(rng, Cout, 8, 8)) if bn else (None, None)
        else:
            x, wT = rng.standard_normal((cells, Cin)).astype(np.float32), rng.standard_normal((Cin, Cout)).astype(np.float32)
            scale, shift = ((rng.uniform(0.5, 2, Cout).astype(np.float32), rng.normal(0, 1, Cout).astype(np.float32))
                            if bn else (None, None))
        out = run_linear_bn(cnt, x, wT, scale, shift)
        ref, S, n = ref_linear_bn(cnt, x, wT, scale, shift)
        if tier == "exact":
            check_exact_tier(S, 2.0 ** -11 * (0.5 if bn else 1.0))
            assert torch.equal(out.double(), ref), f"{Cin}x{Cout} on {cells} cells: {(out.double() != ref).sum()} differ"
        else:
            r = bound_ratio(out, ref, S, n)
            print(f"linear_bn {Cin}x{Cout} on {cells} cells: max |err| / bound = {r:.3g}")
            assert r <= 1.0


# ------------------------------------------------------------------------------------------------------------------------
# pooling between grids, temporal filter, cat_pos, head
# ------------------------------------------------------------------------------------------------------------------------
VW = 8                                   # child voxel: 8 x 8 px; parent voxel 16 x 16 px (cellx = px // 16)
PNX, PNY = 7, 5
CNX, CNY = 2 * PNX, 2 * PNY              # 14 x 10 = 140 cells per sample (a level-3 grid)
PW, PH = CNX * VW, CNY * VW
NC = 100


def sample(seed, C=16, empty=False):
    """one sample's child grid: positions inside its own voxel (so coarse edges join neighbouring parents), features,
    times, CNN head maps [1, C, ny, nx]"""
    rng = np.random.default_rng(seed)
    per = CNX * CNY
    cy, cx = np.divmod(np.arange(per), CNX)
    cnt = ((rng.random(per) < 0.6) * rng.integers(1, 6, per)).astype(np.int32) * (not empty)
    pxy = np.stack([cx * VW + rng.integers(0, VW, per), cy * VW + rng.integers(0, VW, per)], 1).astype(np.int32)
    tmean = rng.choice(np.linspace(0, 1, 17, dtype=np.float32), per)        # ties in t: the filter's strict > matters
    return dict(cnt=cnt, pxy=pxy, mask=rng.integers(0, 512, per).astype(np.int32),
                x=rng.standard_normal((per, C)).astype(np.float32), x128=rng.standard_normal((per, 128)).astype(np.float32),
                tmean=tmean, tmax=np.maximum(tmean, rng.choice(np.linspace(0, 1, 9, dtype=np.float32), per)),
                cls=rng.normal(0, 4, (per, NC + 7)).astype(np.float32), regobj=rng.normal(0, 4, (per, 9)).astype(np.float32),
                add_cls=rng.normal(0, 2, (1, NC, CNY, CNX)).astype(np.float32),
                add_reg=rng.normal(0, 2, (1, 4, CNY, CNX)).astype(np.float32),
                add_obj=rng.normal(0, 2, (1, 1, CNY, CNX)).astype(np.float32))


def batch(samples):
    return {k: np.concatenate([s[k] for s in samples], 0) for k in samples[0]}


def pos_tables():
    inv = lambda n: (1 / torch.Tensor([n]))[0]                                          # noqa: E731
    return (torch.arange(PW).float() * inv(PW)).cuda(), (torch.arange(PH).float() * inv(PH)).cuda()


def run_grid_pool(s, B, aggr, C=16):
    """dagr_grid_pool + _finalize of a [B, CNY, CNX] child grid into [B, PNY, PNX] -> dict of host tensors"""
    from dagr_b200 import _lib
    lib = _lib.load()
    posxr, posyr = pos_tables()
    ch, pa = grid(CNX, CNY, B, PW, PH, posxr, posyr), grid(PNX, PNY, B, PW, PH, posxr, posyr)
    cellx, celly = dev(np.arange(PW, dtype=np.int32) // (2 * VW)), dev(np.arange(PH, dtype=np.int32) // (2 * VW))
    cp = B * PNX * PNY
    acc = torch.zeros(cp * C, dtype=torch.float64, device="cuda")
    accmax, accsum = (acc.view(torch.int32)[:cp * C], None) if aggr == 0 else (None, acc)
    possum = torch.zeros(cp * 3, dtype=torch.float64, device="cuda")
    ptmax, pcnt, pmask, err = (torch.zeros(n, dtype=torch.int32, device="cuda") for n in (cp, cp, cp, 1))
    d = {k: dev(s[k]) for k in ("cnt", "pxy", "tmean", "tmax", "mask", "x")}
    _lib.check(lib.dagr_grid_pool(ch, pa, _lib.ptr(cellx), _lib.ptr(celly), _lib.ptr(d["cnt"]), _lib.ptr(d["pxy"]),
                                  _lib.ptr(d["tmean"]), _lib.ptr(d["tmax"]), _lib.ptr(d["mask"]), _lib.ptr(d["x"]), C, aggr,
                                  _lib.ptr(accmax), _lib.ptr(accsum), _lib.ptr(possum), _lib.ptr(ptmax), _lib.ptr(pcnt),
                                  _lib.ptr(pmask), _lib.ptr(err), _lib.stream_ptr()), "dagr_grid_pool")
    out = dict(pxy=torch.full((cp, 2), -1, dtype=torch.int32, device="cuda"), tmean=torch.full((cp,), np.nan, device="cuda"),
               tmax=torch.full((cp,), np.nan, device="cuda"), x=torch.full((cp, C), np.nan, device="cuda"))
    _lib.check(lib.dagr_grid_pool_finalize(pa, C, aggr, _lib.ptr(accmax), _lib.ptr(accsum), _lib.ptr(possum),
                                           _lib.ptr(ptmax), _lib.ptr(pcnt), _lib.ptr(out["pxy"]), _lib.ptr(out["tmean"]),
                                           _lib.ptr(out["tmax"]), _lib.ptr(out["x"]), _lib.stream_ptr()),
               "dagr_grid_pool_finalize")
    torch.cuda.synchronize()
    out.update(pcnt=pcnt, pmask=pmask, err=err)
    return {k: v.cpu() for k, v in out.items()}


def ref_grid_pool(s, B, aggr):
    """float64 group max / mean of the children of every parent voxel, pooled position through round_to_pixel, the parent
    in-edge bits (self loops dropped)"""
    per, pper = CNX * CNY, PNX * PNY
    cells = np.nonzero(s["cnt"] > 0)[0]
    pcell = s["pxy"] // (2 * VW)                                             # parent (x, y) of every child cell
    P = (cells // per) * pper + pcell[cells, 1] * PNX + pcell[cells, 0]
    cp, C = B * pper, s["x"].shape[1]
    posxr, posyr = (t.cpu().numpy() for t in pos_tables())
    pcnt = np.bincount(P, minlength=cp).astype(np.int32)
    pmask = np.zeros(cp, np.int32)
    for c, p in zip(cells, P):
        cy, cx = divmod(c % per, CNX)
        for bit in range(9):
            sx, sy = cx + bit % 3 - 1, cy + bit // 3 - 1
            if bit == 4 or not (s["mask"][c] >> bit) & 1 or not (0 <= sx < CNX and 0 <= sy < CNY):
                continue
            src = (c // per) * per + sy * CNX + sx
            ddx, ddy = pcell[src] - pcell[c]
            if s["cnt"][src] > 0 and (ddx, ddy) != (0, 0):
                assert abs(ddx) <= 1 and abs(ddy) <= 1
                pmask[p] |= 1 << ((ddy + 1) * 3 + ddx + 1)
    x = np.zeros((cp, C), np.float64)
    pos = np.zeros((cp, 3), np.float64)
    tmax = np.zeros(cp, np.float32)
    for p in np.unique(P):
        kids = cells[P == p]
        x[p] = s["x"][kids].astype(np.float64).max(0) if aggr == 0 else s["x"][kids].astype(np.float64).mean(0)
        pos[p] = np.stack([posxr[s["pxy"][kids, 0]], posyr[s["pxy"][kids, 1]], s["tmean"][kids]], 1).astype(np.float64).mean(0)
        tmax[p] = s["tmean"][kids].max()
    m = torch.from_numpy(pos.astype(np.float32))
    pxy = torch.zeros((cp, 2), dtype=torch.int32)
    for col, size in ((0, PW), (1, PH)):
        q = torch.div(m[:, col] + 1e-5, 1 / torch.Tensor([size]), rounding_mode="floor").clamp(0, size - 1)
        pxy[:, col] = torch.where(torch.from_numpy(pcnt > 0), q.int(), torch.zeros_like(q.int()))
    return dict(pxy=pxy, tmean=m[:, 2], tmax=torch.from_numpy(tmax), x=torch.from_numpy(x.astype(np.float32)),
                pcnt=torch.from_numpy(pcnt), pmask=torch.from_numpy(pmask), err=torch.zeros(1, dtype=torch.int32))


@pytest.mark.parametrize("aggr", [0, 1], ids=["max", "mean"])
def test_grid_pool_vs_float64(aggr):
    """B = 4 with an empty sample; every parent field bit for bit (float64 sums of a few fp32 children are exact)"""
    s = batch([sample(1), sample(2, empty=True), sample(3), sample(4)])
    got, want = run_grid_pool(s, 4, aggr), ref_grid_pool(s, 4, aggr)
    for k in want:
        assert torch.equal(got[k], want[k]), f"{k}: {(got[k] != want[k]).sum()} elements differ"
    assert int(want["pmask"].ne(0).sum()) > 20 and int(want["pcnt"].gt(1).sum()) > 20


def test_grid_pool_flags_a_coarse_edge_over_two_voxels():
    """a child whose neighbour's position lies two parent voxels away sets err_flag (and nothing else changes)"""
    s = sample(1)
    s["cnt"][:] = 0
    c, src = 3 * CNX + 4, 3 * CNX + 5                           # neighbours in x; src's pixel moved 2 parent voxels right
    s["cnt"][[c, src]] = 1
    s["mask"][c] = 1 << 5
    s["pxy"][src, 0] = s["pxy"][c, 0] + 4 * VW
    assert int(run_grid_pool(s, 1, 0)["err"][0]) == 1
    s["pxy"][src, 0] = s["pxy"][c, 0] + 2 * VW
    assert int(run_grid_pool(s, 1, 0)["err"][0]) == 0


def run_head_finish(s, B, a0=13, tail=6, stride=16, nc=NC, maps=True):
    """cls: columns [3, 3 + nc) of a [cells, NC + 7] array; regobj: columns [2, 7) of a [cells, 9] array; the CNN maps
    add_* (maps = False: all three NULL, as in every events-only model); out rows outside [a0, a0 + cells per sample) must
    stay untouched"""
    from dagr_b200 import _lib
    lib = _lib.load()
    per = CNX * CNY
    A = a0 + per + tail
    d = {k: dev(s[k]) for k in ("cnt", "cls", "regobj", "add_reg", "add_obj")}
    d["add_cls"] = dev(s["add_cls"][:, :nc])
    if not maps:
        d["add_cls"] = d["add_reg"] = d["add_obj"] = None
    out = torch.full((B, A, 5 + nc), 7.0, device="cuda")
    out[:, a0:a0 + per] = float("nan")
    _lib.check(lib.dagr_head_finish(grid(CNX, CNY, B), _lib.ptr(d["cnt"]), _lib.ptr(d["cls"][:, 3:]), NC + 7,
                                    _lib.ptr(d["regobj"][:, 2:]), 9, _lib.ptr(d["add_cls"]), _lib.ptr(d["add_reg"]),
                                    _lib.ptr(d["add_obj"]), nc, stride, a0, A, _lib.ptr(out), _lib.stream_ptr()),
               "dagr_head_finish")
    torch.cuda.synchronize()
    return out.cpu()


def test_head_finish_vs_float64_and_torch():
    """nc = 100 on column blocks with CNN maps on every cell (empty cells read 0 + map).  xy exactly as torch fp32;
    exp within CUDA's documented 2 ulp of expf (relative 4u), sigmoid 1 / (1 + expf(-v)) within 6u (4u through the
    quotient, one rounding each for the sum and the division); exp overflow to inf and sigmoid saturation equal torch fp32"""
    head_finish_case(NC, True)


def head_finish_case(nc, maps, B=3, stride=16, a0=13):
    """the checks of test_head_finish_vs_float64_and_torch with nc classes, with the CNN maps or with all three NULL"""
    s = batch([sample(7), sample(8), sample(9)][:B])
    per = CNX * CNY
    # (cell, r, exp overflows or underflows, sigmoid saturates); -20 and -80 are ordinary values far out in the tails
    specials = [(0, 89.0, True, True), (1, 88.7, True, True), (2, 40.0, False, True), (3, -120.0, True, True),
                (4, 120.0, True, True), (5, 20.0, False, True), (6, -20.0, False, False), (7, -80.0, False, False)]
    for i, v, _, _ in specials:                               # on valid cells, with zero maps: r is v itself
        s["cnt"][i] = 1
        s["regobj"][i, 2 + 2:2 + 5] = v
        s["cls"][i, 3:3 + nc] = v
        s["add_reg"][0, 2:, 0, i], s["add_obj"][0, 0, 0, i], s["add_cls"][0, :, 0, i] = 0, 0, 0
    if not maps:
        for k in ("add_cls", "add_reg", "add_obj"):
            s[k] = np.zeros_like(s[k])
    out = run_head_finish(s, B, a0=a0, stride=stride, nc=nc, maps=maps)
    assert (out[:, :a0] == 7).all() and (out[:, a0 + per:] == 7).all()
    o = out[:, a0:a0 + per].reshape(B * per, 5 + nc)
    valid = torch.from_numpy(s["cnt"] > 0)[:, None]
    def col(a, lo, hi):
        return torch.where(valid, torch.from_numpy(a[:, lo:hi]), torch.zeros(1))
    rows = lambda m: torch.from_numpy(np.ascontiguousarray(m)).permute(0, 2, 3, 1).reshape(B * per, -1)     # noqa: E731
    r = col(s["regobj"], 2, 7) + torch.cat([rows(s["add_reg"]), rows(s["add_obj"])], 1)
    v = col(s["cls"], 3, 3 + nc) + rows(s["add_cls"][:, :nc])
    a = torch.arange(B * per) % per
    gy, gx = a // CNX, a % CNX
    assert torch.equal(o[:, 0], (r[:, 0] + gx.float()) * stride) and torch.equal(o[:, 1], (r[:, 1] + gy.float()) * stride)
    e64 = torch.exp(r[:, 2:4].double()) * stride
    sg64 = 1 / (1 + torch.exp(-torch.cat([r[:, 4:5], v], 1).double()))
    got_e, got_s = o[:, 2:4].double(), o[:, 4:].double()
    fin = (e64 < 3.0e38) & (e64 > 2.0e-37)                   # normal fp32 results
    re = ((got_e - e64).abs() / (U * e64))[fin]
    rs = ((got_s - sg64).abs() / (U * sg64))[sg64 > 1.2e-38]
    print(f"head_finish: exp {re.max():.3g} u (bound 4), sigmoid {rs.max():.3g} u (bound 6)")
    assert re.max() <= 4, f"exp: {re.max():.3g} u"
    assert rs.max() <= 6, f"sigmoid: {rs.max():.3g} u"
    assert not torch.isnan(o).any()
    for i, val, e_edge, s_edge in specials:                   # overflow, underflow, saturation: the bits of torch fp32
        t = torch.tensor(val, dtype=torch.float32)
        if e_edge:
            assert torch.equal(o[i, 2:4], (torch.exp(t) * stride).expand(2)), (val, o[i, 2:4])
        if s_edge:
            assert (o[i, 4:] == torch.sigmoid(t)).all(), (val, o[i, 4].item(), torch.sigmoid(t).item())


# ------------------------------------------------------------------------------------------------------------------------
# a sample's rows do not depend on the batch
# ------------------------------------------------------------------------------------------------------------------------
def run_chain(s, B, b):
    """every coarse kernel on the batch s (sample of interest in slot b) -> its rows of each output, grid-conv instances"""
    from dagr_b200 import _lib
    lib = _lib.load()
    per, pper = CNX * CNY, PNX * PNY
    rows = slice(b * per, (b + 1) * per)
    posxr, posyr = pos_tables()
    gr = grid(CNX, CNY, B, PW, PH, posxr, posyr)
    cells = B * per
    cnt, pxy, x = dev(s["cnt"]), dev(s["pxy"]), dev(s["x"])
    res, seen = {}, {}
    xin = torch.full((cells, 18), float("nan"), device="cuda")
    _lib.check(lib.dagr_grid_cat_pos(gr, _lib.ptr(cnt), _lib.ptr(pxy), _lib.ptr(x), 16, _lib.ptr(xin), _lib.stream_ptr()),
               "dagr_grid_cat_pos")
    res["cat_pos"] = xin[rows].cpu()
    wrng = np.random.default_rng(77)                          # the same weights at every B
    for Cin, Cout, src in ((18, 64, xin), (128, 256, dev(s["x128"])), (16, 6400, x)):
        p, _ = conv_params(wrng, "realistic", cells, Cin, Cout, ("bias", "scale", "relu"))
        g = dict(nx=CNX, ny=CNY, B=B, cnt=s["cnt"], pxy=s["pxy"], mask=s["mask"], den_x=real_den()[0], den_y=real_den()[1])
        out, inst = run_grid_conv(g, src.cpu(), 0, 0, Cin, Cout, p)
        res[f"conv{Cin}x{Cout}"], seen[(Cin, Cout)] = out[rows], inst
    wT = torch.from_numpy(wrng.standard_normal((18, 64)).astype(np.float32)).cuda()
    sc, sh = (torch.from_numpy(wrng.standard_normal(64).astype(np.float32)).cuda() for _ in range(2))
    lb = torch.full((cells, 64), float("nan"), device="cuda")
    _lib.check(lib.dagr_grid_linear_bn(cells, _lib.ptr(cnt), _lib.ptr(xin), 18, 64, _lib.ptr(wT), _lib.ptr(sc), _lib.ptr(sh),
                                       _lib.ptr(lb), _lib.stream_ptr()), "dagr_grid_linear_bn")
    res["linear_bn"] = lb[rows].cpu()
    for aggr in (0, 1):
        pool = run_grid_pool(s, B, aggr)
        for k, v in pool.items():
            if k != "err":
                res[f"pool{aggr}_{k}"] = v[b * pper:(b + 1) * pper]
    mask = dev(s["mask"].copy())
    _lib.check(lib.dagr_grid_temporal_filter(gr, _lib.ptr(cnt), _lib.ptr(dev(s["tmax"])), _lib.ptr(mask), _lib.stream_ptr()),
               "dagr_grid_temporal_filter")
    res["temporal_filter"] = mask[rows].cpu()
    res["head_finish"] = run_head_finish(s, B)[b]
    torch.cuda.synchronize()
    return res, seen


@pytest.mark.parametrize("B", [2, 17, 31, 127])
def test_sample_rows_do_not_depend_on_the_batch(B):
    """one sample in slot b of a batch of other samples == the sample at B = 1, bit for bit, in every kernel; the batch
    sizes move dagr_grid_conv through <1>, <4> and <16> (k_grid_conv at 16 -> 6400 throughout)"""
    nsm = n_sm()
    b = B - 1 if B in (2, 31) else B // 2
    one, seen1 = run_chain(batch([sample(1000)]), 1, 0)
    many, seen = run_chain(batch([sample(1000) if i == b else sample(2000 + i) for i in range(B)]), B, b)
    for (Cin, Cout), inst in list(seen1.items()) + list(seen.items()):
        assert len(inst) == 1
    assert seen[(18, 64)] == {instance(18, 64, B * CNX * CNY, nsm)} and seen[(16, 6400)] == {"v1"}
    print(f"B = {B}: instances {seen} (B = 1: {seen1})")
    for k in one:
        assert torch.equal(one[k], many[k]), f"{k}: slot {b} of B = {B} differs from B = 1 in {(one[k] != many[k]).sum()} elements"
