"""The image-sampling kernels' float64 reference, checked without a GPU.

tests/test_image_kernels_gpu.py calls dagr_sample_features, dagr_l1_x0_image and dagr_voxel_sample_max in every form (plain,
_live, _planes, _inc; fp32 NCHW and bf16 NHWC maps) and compares them with the helpers below:
  * bilin_coords: the kernels' fp32 set-up (bilin_setup in image_l1.cu, k_sample_features in coarse.cu), restated with numpy
    float32 operations.  numpy's float32 + - * / are correctly rounded and each is rounded on its own, as the __f*_rn
    intrinsics are, so these are the kernels' exact coordinates: the normalised (gx, gy, gz) -- gz with the batch size
    clamped to 2 when Bi = 1 (net.py:193-221) -- then (ix, iy, iz), their floors and the fractions (tx, ty, tz);
  * ref_sample: trilinear interpolation in float64 at those coordinates, taps outside [0, Bi) x [0, h) x [0, w) skipped
    (zero padding), weights (1 - t) / t in float64.  It also returns S = sum |v_tap| * w_tap for the error bound;
  * ref_voxel / ref_voxel_inc: the per-voxel max or mean of the samples over the voxel's events, and the incremental form
    max(persist, max over the events with arrival index >= min_idx);
  * vs_window: the per-voxel window and path choice of k_voxel_sample_max (fast, general or global), restated from the
    voxel's corner pixels and the header's DAGR_VS_SMEM_FLOATS.

Error bound.  Every output element must satisfy |out - ref| <= c u S + 2 u |ref| (u = 2^-24), c from the operation count of
one sample, worst case and first order in u: the weight wx * wy * wz rounds the three (1 - t) and its two products (5 u),
and the eight taps are accumulated by fp32 FMAs, one rounding each (8 u): C_SAMPLE = 13.  A per-voxel max is exact, so it
keeps the bound of its samples (S of the largest-S event); a mean of n samples adds n additions and the division, over
the mean of S.
"""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
U = 2.0 ** -24
F = np.float32

C_SAMPLE = 5 + 8
FAST, GENERAL, GLOBAL = 0, 1, 2


def vs_cap():
    """DAGR_VS_SMEM_FLOATS of include/dagr_b200.h"""
    text = (ROOT / "include" / "dagr_b200.h").read_text()
    return int(re.search(r"#define DAGR_VS_SMEM_FLOATS\s+(\d+)", text).group(1))


# ------------------------------------------------------------------------------------------------------------------------
# coordinates
# ------------------------------------------------------------------------------------------------------------------------
def split(ix, iy, iz):
    """integer corners and fractions of unnormalised positions, in the positions' own precision (ix - floor(ix) as the
    kernels compute it)"""
    out = {}
    for k, v in (("x", ix), ("y", iy), ("z", iz)):
        f = np.floor(v)
        out[k + "0"] = f.astype(np.int64)
        out["t" + k] = v - f
    return out


def bilin_coords(posx, posy, b, W, H, Bi, h, w):
    """the kernels' fp32 set-up of one (x, y, batch) position per element: normalise with the event resolution (W, H), as
    _sample_features does, unnormalise with the map size as grid_sample(align_corners=True).  Returns the normalised grid
    (gx, gy, gz), the unnormalised (ix, iy, iz) and split()'s corners and fractions, all float32 bits."""
    posx, posy = np.asarray(posx, F), np.asarray(posy, F)
    b = np.broadcast_to(np.asarray(b), posx.shape).astype(F)
    width, height, bs = F(W), F(H), F(Bi if Bi > 1 else 2)
    gx = (F(2) * (posx * width)) / (width - F(1)) - F(1)
    gy = (F(2) * (posy * height)) / (height - F(1)) - F(1)
    gz = (F(2) * b) / (bs - F(1)) - F(1)
    ix = ((gx + F(1)) * F(0.5)) * F(w - 1)
    iy = ((gy + F(1)) * F(0.5)) * F(h - 1)
    iz = ((gz + F(1)) * F(0.5)) * F(Bi - 1)
    co = dict(gx=gx, gy=gy, gz=gz, ix=ix, iy=iy, iz=iz)
    co.update(split(ix, iy, iz))
    return co


def event_coords(geom, x, y, b, Bi, h, w):
    """bilin_coords of events at integer pixels (x, y) of sample b: the kernels read x / W and y / H from geom.posx0 / posy0"""
    px = geom.posx0.cpu().numpy()[np.asarray(x)]
    py = geom.posy0.cpu().numpy()[np.asarray(y)]
    return bilin_coords(px, py, b, geom.W, geom.H, Bi, h, w)


# ------------------------------------------------------------------------------------------------------------------------
# float64 sampling
# ------------------------------------------------------------------------------------------------------------------------
def ref_sample(map64, co):
    """trilinear samples of map64 float64 [Bi, C, h, w] at the coordinates co (split() keys) -> (value, S) float64 [n, C]"""
    m = np.ascontiguousarray(np.asarray(map64, np.float64).transpose(0, 2, 3, 1))          # [Bi, h, w, C]
    Bi, h, w, Cc = m.shape
    n = len(co["x0"])
    val, S = np.zeros((n, Cc)), np.zeros((n, Cc))
    t = {k: np.asarray(co["t" + k], np.float64) for k in "xyz"}
    for dz in (0, 1):
        z = co["z0"] + dz
        wz = t["z"] if dz else 1.0 - t["z"]
        for dy in (0, 1):
            y = co["y0"] + dy
            wy = t["y"] if dy else 1.0 - t["y"]
            for dx in (0, 1):
                x = co["x0"] + dx
                wx = t["x"] if dx else 1.0 - t["x"]
                ok = (z >= 0) & (z < Bi) & (y >= 0) & (y < h) & (x >= 0) & (x < w)
                wgt = np.where(ok, wx * wy * wz, 0.0)[:, None]
                v = m[np.clip(z, 0, Bi - 1), np.clip(y, 0, h - 1), np.clip(x, 0, w - 1)]
                val += v * wgt
                S += np.abs(v) * wgt
    return val, S


def ref_voxel(val, S, cell, cells, mean=False, take=None):
    """per-voxel max or mean of the per-event samples val [n, C] over the events of each voxel (cell [n]; take [n] bool
    selects the events that count) -> (ref, S, c) [cells, C]: S and c so that c u S + 2 u |ref| bounds the voxel's result.
    Voxels without events give 0."""
    n, Cc = val.shape
    take = np.ones(n, bool) if take is None else np.asarray(take, bool)
    cell = np.asarray(cell, np.int64)[take]
    val, S = val[take], S[take]
    cnt = np.bincount(cell, minlength=cells)
    idx = torch.from_numpy(cell)[:, None].expand(-1, Cc)
    if mean:
        k = np.maximum(cnt, 1)[:, None]
        ref = np.zeros((cells, Cc))
        np.add.at(ref, cell, val)
        Sv = np.zeros((cells, Cc))
        np.add.at(Sv, cell, S)
        c = (C_SAMPLE + cnt + 1).astype(np.float64)[:, None] * np.ones((1, Cc))
        return ref / k, Sv / k, c
    ref = torch.full((cells, Cc), -np.inf, dtype=torch.float64).scatter_reduce(0, idx, torch.from_numpy(val), "amax").numpy()
    Sv = torch.zeros((cells, Cc), dtype=torch.float64).scatter_reduce(0, idx, torch.from_numpy(S), "amax").numpy()
    ref[cnt == 0] = 0.0
    return ref, Sv, np.full((cells, Cc), float(C_SAMPLE))


def ref_voxel_inc(val, S, cell, cells, arrival, min_idx, persist):
    """dagr_voxel_sample_max_inc: (xg, persist after the step, S, c).  min_idx = 0: the plain max, persist seeded with it and
    -inf for empty voxels; min_idx > 0: max(persist, the max over the events with arrival index >= min_idx), a copy of persist
    for voxels without such events."""
    cnt_all = np.bincount(np.asarray(cell, np.int64), minlength=cells)
    if min_idx <= 0:
        ref, Sv, c = ref_voxel(val, S, cell, cells)
        new_persist = np.where((cnt_all == 0)[:, None], -np.inf, ref)
        return ref, new_persist, Sv, c
    take = np.asarray(arrival) >= min_idx
    ref, Sv, c = ref_voxel(val, S, cell, cells, take=take)
    has = np.bincount(np.asarray(cell, np.int64)[take], minlength=cells) > 0
    p = np.asarray(persist, np.float64)
    out = np.where(has[:, None], np.maximum(ref, p), p)
    Sv = np.where(has[:, None], Sv, 0.0)                # |max(a', p) - max(a, p)| <= |a' - a|; a copied persist is exact
    empty = cnt_all == 0
    xg = out.copy()
    new_persist = out.copy()
    xg[empty], new_persist[empty] = 0.0, p[empty]
    return xg, new_persist, Sv, c


# ------------------------------------------------------------------------------------------------------------------------
# the voxel kernel's window and path
# ------------------------------------------------------------------------------------------------------------------------
def vs_window(geom, C_, h, w, planes=False, cap=None):
    """k_voxel_sample_max's choice per pool1 voxel (cell order b, cy, cx): the window (pz, ph, pw) of the map its events can
    touch, from the bilin_coords of its first and last pixel in x and y (the coordinates are monotone in both), and the path
    -- FAST (staged, C in {8, 16, 32, 64, 128}), GENERAL (staged, any other C) or GLOBAL (the window exceeds the capacity)."""
    cap = vs_cap() if cap is None else cap
    B, nx, ny = geom.B, geom.nx1, geom.ny1
    vx0, vy0 = geom.vx0.cpu().numpy().astype(np.int64), geom.vy0.cpu().numpy().astype(np.int64)
    b, cy, cx = (a.ravel() for a in np.meshgrid(np.arange(B), np.arange(ny), np.arange(nx), indexing="ij"))
    Bi, bz = (1, np.zeros_like(b)) if planes else (B, b)
    lo = event_coords(geom, vx0[cx], vy0[cy], bz, Bi, h, w)
    hi = event_coords(geom, vx0[cx + 1] - 1, vy0[cy + 1] - 1, bz, Bi, h, w)
    xb, yb, zb = np.maximum(lo["x0"], 0), np.maximum(lo["y0"], 0), np.maximum(lo["z0"], 0)
    xe, ye, ze = np.minimum(hi["x0"] + 1, w - 1), np.minimum(hi["y0"] + 1, h - 1), np.minimum(lo["z0"] + 1, Bi - 1)
    pw, ph, pz = xe - xb + 1, ye - yb + 1, ze - zb + 1
    staged = (pw > 0) & (ph > 0) & (pz > 0) & (pz * ph * pw * C_ <= cap)
    lpe = C_ >> 3
    fast_c = C_ % 8 == 0 and C_ <= 128 and lpe >= 1 and (lpe & (lpe - 1)) == 0
    path = np.where(staged, FAST if fast_c else GENERAL, GLOBAL)
    return path, np.stack([pz, ph, pw], 1)


# ------------------------------------------------------------------------------------------------------------------------
# tests of the reference
# ------------------------------------------------------------------------------------------------------------------------
def _positions(rng, n):
    """normalised positions on the sensor, on its border, up to a pixel outside it and far outside it"""
    px, py = rng.uniform(0, 1, n).astype(F), rng.uniform(0, 1, n).astype(F)
    edge = np.array([0.0, 1.0, -0.004, 1.004, -0.5, 1.7, 0.5, 0.999], F)
    px[:64], py[:64] = np.tile(edge, 8), np.repeat(edge, 8)
    return px, py


@pytest.mark.parametrize("Bi,C_,h,w,W,H", [(1, 5, 7, 9, 240, 180), (3, 4, 15, 21, 240, 180), (6, 3, 1, 13, 640, 480),
                                            (7, 2, 11, 1, 346, 260)])
def test_reference_equals_float64_grid_sample_on_the_same_grid(Bi, C_, h, w, W, H):
    rng = np.random.default_rng(Bi * 100 + C_)
    n = 700
    px, py = _positions(rng, n)
    b = rng.integers(0, Bi, n)
    co = bilin_coords(px, py, b, W, H, Bi, h, w)
    g = np.stack([co["gx"], co["gy"], co["gz"]], 1).astype(np.float64)
    # grid_sample's own unnormalisation, in float64
    ix, iy, iz = ((g[:, 0] + 1) / 2) * (w - 1), ((g[:, 1] + 1) / 2) * (h - 1), ((g[:, 2] + 1) / 2) * (Bi - 1)
    m = rng.standard_normal((Bi, C_, h, w))
    val, S = ref_sample(m, split(ix, iy, iz))
    inp = torch.from_numpy(m).permute(1, 0, 2, 3).unsqueeze(0)                               # [1, C, Bi, h, w]
    gs = torch.nn.functional.grid_sample(inp, torch.from_numpy(g).view(1, 1, 1, n, 3), mode="bilinear", align_corners=True)
    want = gs.view(C_, n).t().numpy()
    assert np.abs(val - want).max() <= 1e-13 * max(1.0, float(S.max())), np.abs(val - want).max()
    assert (S >= np.abs(val) - 1e-12).all()
    # far outside the map every tap is padding (a map of width or height 1 samples its one column / row everywhere)
    far = ((np.abs(px - 0.5) > 0.6) & (w > 1)) | ((np.abs(py - 0.5) > 0.6) & (h > 1))
    assert far.sum() > 0 and (val[far] == 0).all()


@pytest.mark.parametrize("Bi,C_,h,w,W,H", [(1, 16, 45, 60, 240, 180), (2, 8, 27, 41, 640, 480), (6, 4, 9, 13, 320, 215),
                                            (7, 4, 12, 16, 240, 180)])
def test_reference_equals_the_oracle_sample_features_within_the_bound(Bi, C_, h, w, W, H):
    """oracle.ref_ops.sample_features runs torch's fp32 grid_sample on the same normalisation: within the kernels' bound"""
    from oracle.ref_ops import sample_features
    rng = np.random.default_rng(Bi * 10 + C_)
    n = 900
    px, py = _positions(rng, n)
    b = rng.integers(0, Bi, n)
    m = rng.standard_normal((Bi, C_, h, w)).astype(F)
    val, S = ref_sample(m.astype(np.float64), bilin_coords(px, py, b, W, H, Bi, h, w))
    pos = torch.from_numpy(np.stack([px, py], 1))
    got = sample_features(pos, torch.from_numpy(b), torch.from_numpy(m), W, H).double().numpy()
    err = np.abs(got - val)
    bound = C_SAMPLE * U * S + 2 * U * np.abs(val)
    assert (err <= bound).all(), float((err / np.maximum(bound, 1e-300)).max())


def test_reference_is_exact_on_a_linear_map():
    """trilinear interpolation reproduces a map linear in (x, y, z) wherever all 8 taps lie inside it"""
    rng = np.random.default_rng(3)
    Bi, C_, h, w, W, H = 4, 3, 23, 31, 640, 480
    a, kx, ky, kz = (rng.standard_normal(C_) for _ in range(4))
    z, y, x = np.meshgrid(np.arange(Bi), np.arange(h), np.arange(w), indexing="ij")
    m = a[None, :, None, None] + kx[None, :, None, None] * x[:, None] + ky[None, :, None, None] * y[:, None] \
        + kz[None, :, None, None] * z[:, None]
    n = 2000
    px, py = _positions(rng, n)
    b = rng.integers(0, Bi, n)
    co = bilin_coords(px, py, 0.0, W, H, Bi, h, w)
    co["z0"], co["tz"] = np.minimum(b, Bi - 2), np.where(b == Bi - 1, 1.0, rng.uniform(0, 1, n))       # any depth in [0, Bi - 1]
    val, _ = ref_sample(m, co)
    inside = (co["x0"] >= 0) & (co["x0"] + 1 < w) & (co["y0"] >= 0) & (co["y0"] + 1 < h)
    assert inside.sum() > n // 2
    X = co["x0"] + co["tx"].astype(np.float64)
    Y = co["y0"] + co["ty"].astype(np.float64)
    Z = co["z0"] + co["tz"]
    lin = a + kx * X[:, None] + ky * Y[:, None] + kz * Z[:, None]
    assert np.abs(val[inside] - lin[inside]).max() < 1e-12


def test_depth_coordinate_table():
    """fp32 iz = ((2b / (B - 1) - 1) + 1) * 0.5 * (B - 1) is an integer for every sample at B <= 5; sample 1 lands one ulp
    below 1 at B = 6 and one above at B = 7, so it takes a weight of about 1e-7 from plane 0 (B = 6) or plane 2 (B = 7)"""
    for B in range(1, 8):
        co = bilin_coords(np.zeros(B, F), np.zeros(B, F), np.arange(B), 240, 180, B, 5, 5)
        frac = co["iz"].astype(np.float64) - np.arange(B)
        mixing = np.nonzero(frac != 0)[0].tolist()
        if B <= 5:
            assert mixing == [], (B, frac)
        else:
            assert mixing == [1], (B, frac)
    co6 = bilin_coords(F(0), F(0), 1, 240, 180, 6, 5, 5)
    co7 = bilin_coords(F(0), F(0), 1, 240, 180, 7, 5, 5)
    assert (co6["z0"], 1 - float(co6["tz"])) == (0, 2.0 ** -24) and (co7["z0"], float(co7["tz"])) == (1, 2.0 ** -23)


def test_bilin_coords_are_the_fp32_steps():
    """spot values: x / W = 0.5 on a 240-px sensor and a 21-px map lands at ix = fl(fl(fl(240/239) * 0.5) * 20)"""
    co = bilin_coords(F(0.5), F(0.0), 0, 240, 180, 1, 15, 21)
    gx = F(F(240) / F(239)) - F(1)
    assert co["gx"] == gx and co["ix"] == F(F(F(gx + F(1)) * F(0.5)) * F(20))
    assert co["x0"] == 10 and co["tx"] == co["ix"] - F(10) and co["tx"] > 0
    assert co["iy"] == 0 and co["iz"] == 0 and co["gz"] == -1


def test_voxel_reference_max_mean_and_incremental():
    val = np.array([[1.0, -2.0], [3.0, -5.0], [2.0, 4.0]])
    S = np.abs(val) * 2
    cell = np.array([0, 0, 2])
    ref, Sv, c = ref_voxel(val, S, cell, 4)
    assert ref.tolist() == [[3.0, -2.0], [0, 0], [2.0, 4.0], [0, 0]] and Sv[0].tolist() == [6.0, 10.0]
    assert (c == C_SAMPLE).all()
    ref, Sv, c = ref_voxel(val, S, cell, 4, mean=True)
    assert ref.tolist() == [[2.0, -3.5], [0, 0], [2.0, 4.0], [0, 0]] and Sv[0].tolist() == [4.0, 7.0] and c[0, 0] == C_SAMPLE + 3
    xg, p, _, _ = ref_voxel_inc(val, S, cell, 4, np.array([0, 1, 2]), 0, None)
    assert np.isneginf(p[1]).all() and np.isneginf(p[3]).all() and (xg[1] == 0).all() and p[0].tolist() == [3.0, -2.0]
    persist = np.array([[0.5, 0.5], [7.0, 7.0], [9.0, -9.0], [-1.0, -1.0]])
    xg, p, Sv, _ = ref_voxel_inc(val, S, cell, 4, np.array([0, 1, 2]), 1, persist)
    # voxel 0: only event 1 is new -> max(persist, (3, -5)); voxel 1 empty: xg 0, persist kept; voxel 2: (2, 4) vs persist
    assert xg.tolist() == [[3.0, 0.5], [0, 0], [9.0, 4.0], [0, 0]] and p[1].tolist() == [7.0, 7.0] and p[3].tolist() == [-1.0, -1.0]
    assert Sv[0].tolist() == [6.0, 10.0] and Sv[2].tolist() == [4.0, 8.0] and (Sv[[1, 3]] == 0).all()
    xg, p, _, _ = ref_voxel_inc(val, S, cell, 4, np.array([0, 1, 2]), 3, persist)
    assert np.array_equal(xg[[0, 2]], persist[[0, 2]]), "no new events: persist is copied"


def test_voxel_windows_and_paths():
    """640 x 480 (12 x 12 px voxels): the map scale moves the windows across the capacity; the path follows C"""
    from dagr_b200.geometry import Geometry
    g = Geometry(640, 480, 2, device="cpu")
    cap = vs_cap()
    assert cap == 10240
    path, win = vs_window(g, 64, 60, 80)
    assert (path == FAST).all() and (win[:, 0] == np.repeat([2, 1], g.cells1 // 2)).all(), "pz = 2 but for the last sample"
    assert (win[:, 1:] >= 2).all() and (win[:, 1:] <= 4).all()
    path, _ = vs_window(g, 48, 60, 80)
    assert (path == GENERAL).all()
    path, win = vs_window(g, 64, 480, 640)
    # a map at the sensor's size: 11- and 12-pixel voxels touch 11 to 14 map pixels per axis; two planes never fit
    assert (win[:, 1:] >= 11).all() and (win[:, 1:] <= 14).all() and (path[win[:, 0] == 2] == GLOBAL).all()
    path, win = vs_window(g, 64, 480, 640, planes=True)
    assert (win[:, 0] == 1).all()
    # C = 128 on a 92 x 394 map: windows of exactly the capacity stay staged, one column more goes to global memory
    path, win = vs_window(g, 128, 92, 394)
    at, over = (win == [2, 5, 8]).all(1), (win == [2, 5, 9]).all(1)
    assert 2 * 5 * 8 * 128 == cap and at.sum() > 100 and over.sum() > 50
    assert (path[at] == FAST).all() and (path[over] == GLOBAL).all()


def test_header_publishes_the_voxel_staging_capacity():
    src = (ROOT / "dagr_b200" / "csrc" / "image_l1.cu").read_text()
    assert not re.search(r"#define VS_SMEM_FLOATS", src) and "DAGR_VS_SMEM_FLOATS" in src
    assert vs_cap() == 10240
