"""The image-sampling kernels on their own, on synthetic event streams and maps, through the C-ABI.

dagr_sample_features (plain, _planes), dagr_l1_x0_image (plain, _live, _planes) and dagr_voxel_sample_max (plain max and mean,
_planes max and mean, _inc at min_idx = 0 and then > 0), each on fp32 NCHW and bf16 NHWC maps, against the float64 reference of
tests/test_image_kernels_cpu.py: trilinear samples at the kernels' own fp32 coordinates, per element |out - ref| <= c u S +
2 u |ref| (the largest ratio of each case is printed).  The maps hold random bf16 values: their float64 upcast is the
reference of both formats.

Events are sorted on the device (tests.test_l1_kernels_gpu.Stream: border events, clusters, empty samples).  Batch sizes 6
and 7 hold the samples whose fp32 depth coordinate is not an integer (sample 1 takes a weight of about 1e-7 from plane 0 or
plane 2); those neighbouring planes are scaled by 1e6, so a kernel that drops the weight is off by about 0.1.  The voxel cases
restate the kernel's per-voxel path (fast, general, global) from the header's DAGR_VS_SMEM_FLOATS and assert that every
path a case targets holds voxels, windows of exactly the capacity and of one step more included.

A bits tier across kernels: every x0 row equals dagr_sample_features (C = 16) at the event, and the voxel max on all three
paths equals the per-voxel max of dagr_sample_features at the voxel's events, bit for bit (the same tap order and fp32
arithmetic in every kernel).
"""
import ctypes as C
from functools import lru_cache

import numpy as np
import pytest
import torch

from tests.test_image_kernels_cpu import (C_SAMPLE, FAST, GENERAL, GLOBAL, bilin_coords, event_coords, ref_sample, ref_voxel,
                                          ref_voxel_inc, vs_cap, vs_window)
from tests.test_l1_kernels_cpu import bound_ratio, xa_unpack
from tests.test_l1_kernels_gpu import Stream

pytestmark = pytest.mark.gpu

NAN = float("nan")
PATH_NAMES = {FAST: "fast", GENERAL: "general", GLOBAL: "global"}


def _lib():
    from dagr_b200 import _lib as L
    return L, L.load()


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def report(name, r):
    print(f"IMGRATIO {name} {r:.4g}")
    return r


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


def check(name, out, ref, S, c):
    r = report(name, bound_ratio(out, ref, S, c))
    assert r <= 1.0, (name, r)


# ------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------
def depth_scale(B):
    """per-plane scale of the maps: the plane that sample 1 mixes in (B = 6: plane 0, B = 7: plane 2) at 1e6"""
    s = torch.ones(B)
    if B in (6, 7):
        s[0 if B == 6 else 2] = 1e6
    return s


class Map:
    """random bf16 values [n, C, h, w] (times a per-plane scale): the bf16 NHWC tensor, its fp32 NCHW upcast and float64"""

    def __init__(self, seed, n, C_, h, w, scale=None):
        gen = torch.Generator().manual_seed(seed)
        m = torch.rand((n, C_, h, w), generator=gen) * 4 - 2
        if scale is not None:
            m = m * scale.view(-1, 1, 1, 1)
        m = m.to(torch.bfloat16)
        self.bf16 = m.cuda().contiguous(memory_format=torch.channels_last)
        self.f32 = m.float().cuda().contiguous()
        self.f64 = m.double().numpy()
        self.shape = (n, C_, h, w)

    def fmt(self, bf16):
        return self.bf16 if bf16 else self.f32


FORMATS = (False, True)
SFX = {False: "", True: "_bf16"}


def plane_table(B, P_, stride):
    """int32[B * stride]: sample b reads entry b * stride, some of them below 0 and at or above P_ (clamped by the kernels);
    the entries between are junk the kernels must not read"""
    t = torch.full((B * stride,), 99, dtype=torch.int32)
    choice = [-3, P_ + 2, P_ - 1, 0, P_, 1, -1, 2]
    for b in range(B):
        t[b * stride] = choice[b % len(choice)] if b < len(choice) else (3 * b + 1) % P_
    return t, t[::stride][:B].long().clamp(0, P_ - 1)


@lru_cache(maxsize=None)
def stream(name):
    if name == "one":                                                    # a single event on the sensor's last pixel
        b, pos = torch.zeros(1, dtype=torch.int32), torch.tensor([[239, 179, 5]], dtype=torch.int32)
        return Stream(240, 180, 1, 40, 0, events=(b, pos))
    return Stream(**STREAMS[name])


STREAMS = {
    "240_B1": dict(W=240, H=180, B=1, seed=31, n_bg=3001, border=250),
    "320_B2": dict(W=320, H=215, B=2, seed=32, n_bg=2501, border=250, clusters=[(1, 10, 10, 600)]),
    "640_B2": dict(W=640, H=480, B=2, seed=33, n_bg=6001, border=500, clusters=[(0, 20, 20, 800)]),
    "640_B3": dict(W=640, H=480, B=3, seed=34, n_bg=4001, border=250, empty=(1,)),
    "240_B6": dict(W=240, H=180, B=6, seed=35, n_bg=1501, border=250),
    "240_B7": dict(W=240, H=180, B=7, seed=36, n_bg=1201, border=250),
    "one": None,
}


def sorted_events(s):
    """(x, y, b, arrival id, voxel) per sorted position"""
    a = s.perm
    return s.pos[a, 0].numpy(), s.pos[a, 1].numpy(), s.batch[a].long().numpy(), a.numpy(), s.cell_of[a].numpy()


def event_ref(s, mp, planes=None):
    """float64 samples of map mp at every event, sorted order -> (value, S) [N, C].  planes = the clamped plane per sample:
    each sample reads its plane as a batch of one"""
    x, y, b, _, _ = sorted_events(s)
    n, _, h, w = mp.shape
    if planes is None:
        return ref_sample(mp.f64, event_coords(s.geom, x, y, b, n, h, w))
    val, S = np.zeros((s.N, mp.shape[1])), np.zeros((s.N, mp.shape[1]))
    for bb in range(s.geom.B):
        k = b == bb
        if k.any():
            val[k], S[k] = ref_sample(mp.f64[int(planes[bb])][None], event_coords(s.geom, x[k], y[k], 0, 1, h, w))
    return val, S


# ------------------------------------------------------------------------------------------------------------------------
# launches
# ------------------------------------------------------------------------------------------------------------------------
def run_sample(mp, bf16, posx, posy, bidx, W, H, ldo, c0, planes=None):
    L, lib = _lib()
    n_, C_, h, w = mp.shape
    n = posx.shape[0]
    out = torch.full((n, ldo), NAN, device="cuda")
    args = (P(posx), P(posy), P(bidx), n, W, H, P(out), ldo, c0, st())
    if planes is None:
        L.check(getattr(lib, "dagr_sample_features" + SFX[bf16])(P(mp.fmt(bf16)), n_, C_, h, w, *args), "sample_features")
    else:
        tab, stride = planes
        L.check(getattr(lib, "dagr_sample_features_planes" + SFX[bf16])(P(mp.fmt(bf16)), n_, P(tab), stride, C_, h, w, *args),
                "sample_features_planes")
    torch.cuda.synchronize()
    return out.cpu()


def run_x0(s, mp, bf16, form, planes=None, cap=None):
    """form: plain, live (xyb of capacity cap > N with copies of live words behind the live total) or planes"""
    L, lib = _lib()
    n_, _, h, w = mp.shape
    N = s.N if cap is None else cap
    xyb = s.xyb
    if cap is not None:
        xyb = torch.zeros(cap + 1, dtype=torch.int32, device="cuda")
        xyb[:s.N] = s.xyb[:s.N]
        xyb[s.N:cap] = s.xyb[:s.N].repeat(cap // s.N + 1)[:cap - s.N]
    x0 = torch.full((2 * N * 8,), NAN, device="cuda")
    g = C.byref(s.geom.c_geom)
    cw = (16,) if bf16 else ()
    img = P(mp.fmt(bf16))
    if form == "plain":
        L.check(getattr(lib, "dagr_l1_x0_image" + SFX[bf16])(g, N, P(xyb), None, img, *cw, h, w, P(x0), st()), "x0")
    elif form == "live":
        L.check(getattr(lib, "dagr_l1_x0_image_live" + SFX[bf16])(g, N, P(s.start), P(xyb), None, img, *cw, h, w, P(x0), st()), "x0_live")
    else:
        tab, stride = planes
        L.check(getattr(lib, "dagr_l1_x0_image_planes" + SFX[bf16])(g, N, P(s.start), P(xyb), None, img, *cw, h, w, n_, P(tab), stride,
                                                                     P(x0), st()), "x0_planes")
    torch.cuda.synchronize()
    return x0.cpu(), N


def run_voxel(s, mp, bf16, ldx, c0, mean=0, planes=None, inc=None):
    """plain / planes (mean 0 or 1) or inc = (min_idx, persist f32 [cells, C] on the host) -> (xg, persist after)"""
    L, lib = _lib()
    n_, C_, h, w = mp.shape
    xg = torch.full((s.cells, ldx), NAN, device="cuda")
    g = C.byref(s.geom.c_geom)
    img = P(mp.fmt(bf16))
    persist = None
    if inc is not None:
        persist = inc[1].clone().cuda()
        L.check(getattr(lib, "dagr_voxel_sample_max_inc" + SFX[bf16])(g, s.N, P(s.start), P(s.xyb), P(s.ti), img, C_, h, w, inc[0],
                                                                       P(persist), P(xg), ldx, c0, 0, st()), "voxel_inc")
    elif planes is not None:
        tab, stride = planes
        L.check(getattr(lib, "dagr_voxel_sample_max_planes" + SFX[bf16])(g, s.N, P(s.start), P(s.xyb), img, C_, h, w, n_, P(tab), stride,
                                                                          P(xg), ldx, c0, mean, st()), "voxel_planes")
    else:
        L.check(getattr(lib, "dagr_voxel_sample_max" + SFX[bf16])(g, s.N, P(s.start), P(s.xyb), img, C_, h, w, P(xg), ldx, c0, mean,
                                                                    st()), "voxel")
    torch.cuda.synchronize()
    return xg.cpu(), None if persist is None else persist.cpu()


def sentinel_kept(t, c0, C_):
    """columns outside [c0, c0 + C) of a NaN-filled output keep their bits"""
    nan = torch.tensor(NAN).view(torch.int32)
    b = bits(t)
    return bool((b[:, :c0] == nan).all() and (b[:, c0 + C_:] == nan).all())


# ------------------------------------------------------------------------------------------------------------------------
# sample_features
# ------------------------------------------------------------------------------------------------------------------------
SF_CASES = {
    # Bi, C, h, w, sensor W x H, nodes
    "B1_C1": (1, 1, 15, 21, 240, 180, 1001),
    "B2_C3_h1": (2, 3, 1, 37, 640, 480, 1003),
    "B3_C33_w1": (3, 33, 29, 1, 346, 260, 777),
    "B6_C64_mix": (6, 64, 13, 17, 640, 480, 1001),
    "B7_C256_mix": (7, 256, 9, 11, 240, 180, 501),
    "B2_C512_large": (2, 512, 181, 241, 240, 180, 303),
}


def sf_inputs(Bi, W, H, n, seed):
    rng = np.random.default_rng(seed)
    px, py = rng.uniform(0, 1, n).astype(np.float32), rng.uniform(0, 1, n).astype(np.float32)
    # the sensor's corners and edges, up to a pixel outside them (partial padding) and far outside (all padding)
    ex = np.array([0.0, (W - 1) / W, 1.0, -0.5 / W, (W - 0.25) / W, -1.0 / W, -0.7, 1.8], np.float32)
    ey = np.array([0.0, (H - 1) / H, 1.0, -0.5 / H, (H - 0.25) / H, -1.0 / H, -0.7, 1.8], np.float32)
    px[:64], py[:64] = np.tile(ex, 8), np.repeat(ey, 8)
    b = rng.integers(0, Bi, n)
    if Bi in (6, 7):
        b[64:n // 2] = 1                                                  # the mixing sample
    return px, py, b


@pytest.mark.parametrize("name", list(SF_CASES))
def test_sample_features_against_float64_in_every_form(name):
    Bi, C_, h, w, W, H, n = SF_CASES[name]
    assert n % 4
    px, py, b = sf_inputs(Bi, W, H, n, list(SF_CASES).index(name))
    posx, posy = torch.from_numpy(px).cuda(), torch.from_numpy(py).cuda()
    bidx = torch.from_numpy(b.astype(np.int32)).cuda()
    c0, ldo = 7, 7 + C_ + 3
    mp = Map(11, Bi, C_, h, w, depth_scale(Bi))
    co = bilin_coords(px, py, b, W, H, Bi, h, w)
    ref, S = ref_sample(mp.f64, co)
    if h > 1 and w > 1:
        assert (S == 0).sum() >= 8 * C_ and ((S > 0) & ((co["x0"] < 0) | (co["x0"] >= w - 1))[:, None]).any(), "padding cases"
    if Bi in (6, 7):
        mix = b == 1
        assert (co["tz"][mix] != 0).all(), "sample 1 mixes a neighbouring plane"
    P_ = 2 * Bi + 1
    pm = Map(12, P_, C_, h, w)
    tab, pl = plane_table(Bi, P_, 3)
    assert (tab[::3] < 0).any() and (tab[::3] >= P_).any() or Bi < 2
    pref, pS = np.zeros_like(ref), np.zeros_like(ref)
    co1 = bilin_coords(px, py, 0, W, H, 1, h, w)
    for bb in range(Bi):
        k = b == bb
        sub = {key: v[k] for key, v in co1.items()}
        pref[k], pS[k] = ref_sample(pm.f64[int(pl[bb])][None], sub)
    for bf16 in FORMATS:
        f = "bf16" if bf16 else "fp32"
        o = run_sample(mp, bf16, posx, posy, bidx, W, H, ldo, c0)
        assert sentinel_kept(o, c0, C_), (name, f)
        check(f"sample_features/{name}/{f}", o[:, c0:c0 + C_], ref, S, C_SAMPLE)
        o = run_sample(pm, bf16, posx, posy, bidx, W, H, ldo, c0, planes=(tab.cuda(), 3))
        assert sentinel_kept(o, c0, C_), (name, f, "planes")
        check(f"sample_features_planes/{name}/{f}", o[:, c0:c0 + C_], pref, pS, C_SAMPLE)


# ------------------------------------------------------------------------------------------------------------------------
# x0_image
# ------------------------------------------------------------------------------------------------------------------------
X0_CASES = {"240_B1": (45, 60), "320_B2": (54, 81), "640_B3": (120, 160), "240_B6": (23, 31), "240_B7": (17, 29), "one": (5, 7)}


@pytest.mark.parametrize("name", list(X0_CASES))
def test_x0_image_against_float64_in_every_form(name):
    s = stream(name)
    h, w = X0_CASES[name]
    B, N = s.geom.B, s.N
    assert N == 1 or N % 8, "N not a multiple of the swizzle period"
    mp = Map(21, B, 16, h, w, depth_scale(B))
    ref, S = event_ref(s, mp)
    P_ = 2 * B + 1
    pm = Map(22, P_, 16, h, w)
    tab, pl = plane_table(B, P_, 2)
    pref, pS = event_ref(s, pm, planes=pl)
    cap = N + 37
    for bf16 in FORMATS:
        f = "bf16" if bf16 else "fp32"
        for form in ("plain", "live", "planes"):
            x0, NN = run_x0(s, pm if form == "planes" else mp, bf16, form, planes=(tab.cuda(), 2), cap=cap if form == "live" else None)
            rows = xa_unpack(x0, NN)
            if form == "live":
                assert torch.isnan(rows[N:]).all(), "rows at or beyond the live total keep their sentinel"
            rr, ss = (pref, pS) if form == "planes" else (ref, S)
            check(f"x0_{form}/{name}/{f}", rows[:N], rr, ss, C_SAMPLE)
    # bits tier: every x0 row is dagr_sample_features (C = 16) at (posx0[x], posy0[y], b)
    x, y, b, _, _ = sorted_events(s)
    posx = s.geom.posx0.cpu()[torch.from_numpy(x)].contiguous().cuda()
    posy = s.geom.posy0.cpu()[torch.from_numpy(y)].contiguous().cuda()
    sf = run_sample(mp, False, posx, posy, torch.from_numpy(b.astype(np.int32)).cuda(), s.geom.W, s.geom.H, 16, 0)
    x0, _ = run_x0(s, mp, False, "plain")
    assert torch.equal(bits(xa_unpack(x0, N)), bits(sf)), "x0_image and sample_features differ in their bits"


# ------------------------------------------------------------------------------------------------------------------------
# voxel_sample_max
# ------------------------------------------------------------------------------------------------------------------------
VOX_CASES = {
    # stream, C, h, w, the paths the case must reach
    "240_B1_C16": ("240_B1", 16, 45, 60, {FAST}),
    "640_B3_C8_empty": ("640_B3", 8, 60, 80, {FAST}),
    # a map wider than the sensor: two planes never fit, one plane of the 11-pixel voxels does
    "640_B2_C64_global": ("640_B2", 64, 480, 641, {FAST, GLOBAL}),
    "640_B2_C128_capacity": ("640_B2", 128, 92, 394, {FAST, GLOBAL}),
    "320_B2_C24": ("320_B2", 24, 53, 81, {GENERAL}),
    "640_B3_C48": ("640_B3", 48, 27, 41, {GENERAL}),
    "640_B2_C256": ("640_B2", 256, 120, 160, {GENERAL, GLOBAL}),
    "240_B6_C16_mix": ("240_B6", 16, 23, 31, {FAST}),
    "240_B7_C32_mix": ("240_B7", 32, 23, 31, {FAST}),
    "240_B7_C24_mix": ("240_B7", 24, 23, 31, {GENERAL}),
}


def check_voxel(name, xg, ref, S, c, c0, C_, nonempty):
    assert sentinel_kept(xg, c0, C_), name
    out = xg[:, c0:c0 + C_]
    assert (out[~nonempty] == 0).all(), (name, "empty voxels give 0")
    check(name, out, ref, S, c)


@pytest.mark.parametrize("name", list(VOX_CASES))
def test_voxel_sample_max_against_float64_in_every_form(name):
    sname, C_, h, w, targets = VOX_CASES[name]
    s = stream(sname)
    B, cells = s.geom.B, s.cells
    nonempty = torch.from_numpy(s.nown > 0)
    path, win = vs_window(s.geom, C_, h, w)
    ne = nonempty.numpy()
    reached = {PATH_NAMES[k]: int(((path == k) & ne).sum()) for k in (FAST, GENERAL, GLOBAL)}
    print("VOXPATHS", name, reached)
    for k in (FAST, GENERAL, GLOBAL):
        assert (reached[PATH_NAMES[k]] >= 3) == (k in targets), (name, reached)
    vol = win.prod(1) * C_
    if name == "640_B2_C128_capacity":
        cap = vs_cap()
        assert ((vol == cap) & ne).sum() >= 3 and ((win == [2, 5, 8]).all(1) & ne).any(), "windows of exactly the capacity"
        assert ((win == [2, 5, 9]).all(1) & ne).sum() >= 3, "windows of one column more"
    # windows clipped at the map's right and bottom edges, and empty voxels
    last_col = (np.arange(cells) % s.geom.nx1) == s.geom.nx1 - 1
    last_row = ((np.arange(cells) // s.geom.nx1) % s.geom.ny1) == s.geom.ny1 - 1
    assert (last_col & ne).sum() >= 3 and (last_row & ne).sum() >= 3 and (~ne).sum() >= 1, name

    _, _, _, arrival, cell = sorted_events(s)
    mp = Map(31, B, C_, h, w, depth_scale(B))
    val, S = event_ref(s, mp)
    P_ = 2 * B + 1
    pm = Map(32, P_, C_, h, w)
    tab, pl = plane_table(B, P_, 2)
    pval, pS = event_ref(s, pm, planes=pl)
    c0, ldx = 16, 16 + C_ + 5
    m2 = Map(33, B, C_, h, w, depth_scale(B))
    val2, S2 = event_ref(s, m2)
    assert torch.equal(s.ti[:2 * s.N].view(s.N, 2)[:, 1].cpu().long(), s.perm), "ti[p].y is the arrival index"
    min_idx = s.N // 2
    for bf16 in FORMATS:
        f = "bf16" if bf16 else "fp32"
        for mean in (0, 1):
            agg = "mean" if mean else "max"
            xg, _ = run_voxel(s, mp, bf16, ldx, c0, mean)
            check_voxel(f"voxel_{agg}/{name}/{f}", xg, *ref_voxel(val, S, cell, cells, mean=bool(mean)), c0, C_, nonempty)
            xg, _ = run_voxel(s, pm, bf16, ldx, c0, mean, planes=(tab.cuda(), 2))
            check_voxel(f"voxel_planes_{agg}/{name}/{f}", xg, *ref_voxel(pval, pS, cell, cells, mean=bool(mean)), c0, C_, nonempty)
        # incremental: seed (min_idx = 0) on one map, then step (min_idx > 0) on another
        prior = torch.full((cells, C_), 1234.5)
        xg, pers = run_voxel(s, mp, bf16, ldx, c0, inc=(0, prior))
        want_xg, want_p, Sv, c = ref_voxel_inc(val, S, cell, cells, arrival, 0, None)
        check_voxel(f"voxel_inc0/{name}/{f}", xg, want_xg, Sv, c, c0, C_, nonempty)
        assert torch.equal(bits(pers[nonempty]), bits(xg[nonempty, c0:c0 + C_])), "persist is seeded with the result"
        assert torch.isneginf(pers[~nonempty]).all(), "empty voxels seed -inf"
        # a persist with finite values everywhere: empty voxels and voxels without new events must keep them
        seed = torch.where(torch.isneginf(pers), torch.full_like(pers, -7.25), pers)
        xg, pers2 = run_voxel(s, m2, bf16, ldx, c0, inc=(min_idx, seed))
        want_xg, want_p, Sv, c = ref_voxel_inc(val2, S2, cell, cells, arrival, min_idx, seed.double().numpy())
        check_voxel(f"voxel_inc/{name}/{f}", xg, want_xg, Sv, c, c0, C_, nonempty)
        has_new = np.bincount(cell[arrival >= min_idx], minlength=cells) > 0
        untouched = torch.from_numpy(~has_new)
        assert untouched.any() and torch.equal(bits(pers2[untouched]), bits(seed[untouched])), "persist rows without new events"
        kept = untouched & nonempty
        assert torch.equal(bits(xg[kept, c0:c0 + C_]), bits(seed[kept])), "a voxel without new events copies persist"
        assert torch.equal(bits(pers2[~untouched]), bits(xg[~untouched, c0:c0 + C_])), "persist holds the new running max"
        check(f"voxel_inc_persist/{name}/{f}", pers2[torch.from_numpy(has_new)], want_p[has_new], Sv[has_new], c[has_new])

    # bits tier: the voxel max is the per-voxel max of dagr_sample_features at the voxel's events, on every path
    x, y, b, _, _ = sorted_events(s)
    posx = s.geom.posx0.cpu()[torch.from_numpy(x)].contiguous().cuda()
    posy = s.geom.posy0.cpu()[torch.from_numpy(y)].contiguous().cuda()
    sf = run_sample(mp, False, posx, posy, torch.from_numpy(b.astype(np.int32)).cuda(), s.geom.W, s.geom.H, C_, 0)
    idx = torch.from_numpy(cell)[:, None].expand(-1, C_)
    want = torch.full((cells, C_), -np.inf).scatter_reduce(0, idx, sf, "amax")
    want[~nonempty] = 0
    xg, _ = run_voxel(s, mp, False, ldx, c0, 0)
    for k in (FAST, GENERAL, GLOBAL):
        sel = torch.from_numpy((path == k) & ne)
        assert torch.equal(bits(xg[sel, c0:c0 + C_]), bits(want[sel])), (name, PATH_NAMES[k], "differs from sample_features")
