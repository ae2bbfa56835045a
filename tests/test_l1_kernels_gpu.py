"""The event-level kernels on their own, on synthetic event streams, through the C-ABI.

dagr_l1_build_tc (and the fp32 dagr_l1_build), dagr_l1_conv_b_pool_voxel_tc in its three template instances (PLAIN, general,
pool_mean), dagr_l1_conv_a_image_tc / _inc and dagr_xa_permute against the float64 reference of
tests/test_l1_kernels_cpu.py: edges from the graph oracle mapped to sorted positions through the sort's perm (the kernels'
nbr / off / degree slot / cellmask are asserted equal to them bit for bit), oracle.ref_ops.spline_conv on the fp32 basis and
float64 everything else.  Two tiers: exact inputs on dyadic geometries (torch.equal) and realistic ones (per element
|out - ref| <= c u S + 2 u |ref|, c from the operation counts; the largest ratio of each case is printed).

Per-voxel instances are chosen on the device from the 3x3 neighbourhood's node count; the tests restate that choice from the
sort's start table and the header's DAGR_L1_* capacities, assert that every class holds voxels and that the kernels' own
over-capacity counter wl_hdr[0] equals the restated count, so the coverage cannot silently move.  Every node's rows must be
the same bits in every instance (lean / regular / dense, staged / gathered, defer 0 and 1) and in every batch it is part of.
"""
import ctypes as C
from functools import lru_cache

import numpy as np
import pytest
import torch

from tests.test_l1_kernels_cpu import (C_BUILD_FP32, C_BUILD_TC, C_CONV, C_IMAGE, C_SKIP, U, bound_ratio, build_dense_smem_bytes,
                                       degrees, dyadic,
                                       exact_tier_budget, l1_caps, make_events, oracle_edges, ref_conv, voxel_classes,
                                       voxel_stats, xa_pack, xa_unpack)

pytestmark = pytest.mark.gpu

CAPS = l1_caps()
NAN = float("nan")


def _lib():
    from dagr_b200 import _lib as L
    return L, L.load()


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def report(name, r):
    print(f"L1RATIO {name} {r:.4g}")
    return r


def _fill(arr, t):
    a = np.ascontiguousarray(np.asarray(t, np.float32).ravel())
    C.memmove(arr, a.ctypes.data, a.nbytes)


# ------------------------------------------------------------------------------------------------------------------------
# one synthetic stream, sorted on the device, with its oracle graph
# ------------------------------------------------------------------------------------------------------------------------
class Stream:
    def __init__(self, W, H, B, seed, n_bg, radius=0.01, K=16, clusters=(), border=0, empty=(), region=None, events=None, feat=None,
                 time_window=1_000_000, max_queue_size=128, expect_flag=0):
        from dagr_b200.geometry import Geometry
        L, lib = _lib()
        self.geom = geom = Geometry(W, H, B, radius=radius, time_window=time_window, max_neighbors=K, max_queue_size=max_queue_size,
                                    device="cuda")
        if events is None:
            box = []
            for (b, cx, cy, n) in clusters:                     # a cluster fills one pool1 voxel
                x0, x1, y0, y1 = int(geom.vx0[cx]), int(geom.vx0[cx + 1]), int(geom.vy0[cy]), int(geom.vy0[cy + 1])
                box.append((b, x0, y0, x1 - x0, y1 - y0, n))
            batch, pos = make_events(region[0] if region else W, region[1] if region else H, B, n_bg, seed, box, border, empty)
        else:
            batch, pos = events
        self.batch, self.pos = batch, pos
        self.N = N = int(batch.shape[0])
        rng = np.random.default_rng(seed + 1)
        self.feat = torch.from_numpy(rng.choice([-1.0, 1.0], N).astype(np.float32)) if feat is None else feat
        ws = L.EventWs()
        L.check(lib.dagr_event_workspace_bytes(C.byref(geom.c_geom), N, C.byref(ws)), "ws")
        buf = lambda name: torch.zeros(getattr(ws, name) // 4 + 1, dtype=torch.int32, device="cuda")   # noqa: E731
        self.start, self.perm_d, self.ti = buf("start"), buf("perm"), buf("ti")
        self.xyb, self.feat_s = buf("xyb"), torch.zeros(N + 1, device="cuda")
        flags = torch.zeros(4, dtype=torch.int32, device="cuda")
        # every buffer is bound to a name for the whole call: a temporary goes back to the caching allocator as soon as its
        # pointer is taken, and the next one could be handed the same memory
        work = [buf(k) for k in ("key", "tmp", "count", "blocksums")]
        inp = [batch.cuda(), pos.cuda(), self.feat.cuda()]
        L.check(lib.dagr_graph_sort(C.byref(geom.c_geom), *map(P, inp), N, *map(P, work), P(self.start),
                                    P(self.perm_d), P(self.ti), P(self.xyb), P(self.feat_s), P(flags), st()), "sort")
        torch.cuda.synchronize()
        assert int(flags[0]) == expect_flag
        self.flags = flags
        self.perm = self.perm_d[:N].long().cpu()
        self.pos_of = torch.empty(N, dtype=torch.long)
        self.pos_of[self.perm] = torch.arange(N)
        self.nown, self.total = voxel_stats(geom, self.start[:geom.NK + 1].cpu().numpy())
        self.classes = voxel_classes(self.nown, self.total, CAPS)
        bc = batch.clamp(0, B - 1)                              # the sample ids the kernels use (the oracle has no others)
        self.edges = oracle_edges(geom, bc, pos)
        self.deg = degrees(self.edges, N)
        self.cells = geom.cells1
        x, y = pos[:, 0].long(), pos[:, 1].long()
        self.px, self.py = geom.posx0[x], geom.posy0[y]
        lv = geom.levels[0]
        self.cell_of = (bc.long() * geom.ny1 + lv.celly[y].long()) * geom.nx1 + lv.cellx[x].long()   # arrival order

    def ev3(self):
        """(polarity, x / W, y / H) per node, arrival order, float64"""
        return torch.stack([self.feat, self.px, self.py], 1).double()

    def sorted_to_arrival(self, rows):
        return rows[self.pos_of]

    def arrival_to_sorted(self, rows):
        return rows[self.perm]

    def expected_adjacency(self):
        """(nbr, off) int64 [16, N] in sorted positions (-1 where no slot), degree per sorted position, cellmask per voxel"""
        N, g = self.N, self.geom
        src, dst = self.edges
        m = src != dst
        src, dst = src[m], dst[m]
        first = torch.zeros(N + 1, dtype=torch.long)
        first[1:] = torch.cumsum(torch.bincount(dst, minlength=N), 0)
        slot = torch.arange(len(dst)) - first[dst]
        R = 2 * g.r + 1
        cell_idx = torch.full((R * R,), -1, dtype=torch.long)
        sp = g.spiral.long()
        cell_idx[(sp[:, 0] + g.r) * R + sp[:, 1] + g.r] = torch.arange(g.ncell)
        d = self.pos[src, :2].long() - self.pos[dst, :2].long()
        nbr = torch.full((16, N), -1, dtype=torch.long)
        off = torch.full((16, N), -1, dtype=torch.long)
        nbr[slot, self.pos_of[dst]] = self.pos_of[src]
        off[slot, self.pos_of[dst]] = cell_idx[(d[:, 0] + g.r) * R + d[:, 1] + g.r]
        deg = torch.zeros(N, dtype=torch.long)
        deg[self.pos_of] = self.deg
        lv = g.levels[0]
        cs, cd = self.cell_of[src], self.cell_of[dst]
        xs, ys = lv.cellx[self.pos[src, 0].long()].long(), lv.celly[self.pos[src, 1].long()].long()
        xd, yd = lv.cellx[self.pos[dst, 0].long()].long(), lv.celly[self.pos[dst, 1].long()].long()
        bit = (ys - yd + 1) * 3 + (xs - xd + 1)
        mask = np.zeros(self.cells, np.int64)
        keep = (bit != 4).numpy()
        np.bitwise_or.at(mask, cd.numpy()[keep], (1 << bit.numpy()[keep]))
        assert ((cs == cd) | (bit != 4)).all()
        return nbr, off, deg, torch.from_numpy(mask), (src, dst)


def new_mask(s, min_idx):
    """cellmask bits contributed by the edges of nodes with arrival index >= min_idx"""
    _, _, _, _, (src, dst) = s.expected_adjacency()
    lv = s.geom.levels[0]
    xs, ys = lv.cellx[s.pos[src, 0].long()].long(), lv.celly[s.pos[src, 1].long()].long()
    xd, yd = lv.cellx[s.pos[dst, 0].long()].long(), lv.celly[s.pos[dst, 1].long()].long()
    bit = ((ys - yd + 1) * 3 + (xs - xd + 1)).numpy()
    keep = (bit != 4) & (dst >= min_idx).numpy()
    mask = np.zeros(s.cells, np.int64)
    np.bitwise_or.at(mask, s.cell_of[dst].numpy()[keep], 1 << bit[keep])
    return torch.from_numpy(mask)


# ------------------------------------------------------------------------------------------------------------------------
# parameters of the two tiers
# ------------------------------------------------------------------------------------------------------------------------
def nonzero_scale(rng):
    """exact-tier BN scales: {-1, -1/2, 1/2, 1}, never zero, so that the bit-exact comparison sees every channel"""
    return rng.choice(np.array([-1.0, -0.5, 0.5, 1.0], np.float32), 16)


def build_params(rng, exact, pol_zero=False):
    """conv_a 3 -> 16: w [15, 3, 16], root [3, 16], folded BN"""
    if exact:
        w, root = dyadic(rng, (15, 3, 16), 2, 1), dyadic(rng, (3, 16), 2, 1)
        if pol_zero:
            w[:, 0], root[0] = 0, 0
        scale, shift = nonzero_scale(rng), dyadic(rng, 16, 4, 4)
    else:
        w, root = (rng.standard_normal((15, 3, 16)) * 0.4).astype(np.float32), (rng.standard_normal((3, 16)) * 0.4).astype(np.float32)
        scale, shift = (rng.uniform(0.5, 2.0, 16) * rng.choice([-1, 1], 16)).astype(np.float32), (rng.standard_normal(16) * 0.3).astype(np.float32)
    return dict(w=w, root=root, scale=scale, shift=shift)


def conv_params(rng, exact, cin=16):
    """conv 16 -> 16 (+ the skip rows), folded BN of the conv and of the skip branch"""
    if exact:
        w, root = dyadic(rng, (15, cin, 16), 3, 2), dyadic(rng, (cin, 16), 3, 2)
        skip = dyadic(rng, (19, 16), 3, 2)
        scale, shift = nonzero_scale(rng), dyadic(rng, 16, 4, 4)
        sscale, sshift = nonzero_scale(rng), dyadic(rng, 16, 4, 4)
    else:
        n = lambda *s: (rng.standard_normal(s) * 0.25).astype(np.float32)            # noqa: E731
        w, root, skip = n(15, cin, 16), n(cin, 16), n(19, 16)                 # skip rows 16..18: polarity, x, y
        scale = (rng.uniform(0.5, 2.0, 16) * rng.choice([-1, 1], 16)).astype(np.float32)
        sscale = rng.uniform(0.5, 2.0, 16).astype(np.float32)
        shift, sshift = n(16), n(16)
    return dict(w=w, root=root, skip=skip, scale=scale, shift=shift, sscale=sscale, sshift=sshift)


def node_rows(rng, N, exact, bits=4):
    return torch.from_numpy(dyadic(rng, (N, 16), bits, 2) if exact else rng.standard_normal((N, 16)).astype(np.float32))


# ------------------------------------------------------------------------------------------------------------------------
# kernel launches
# ------------------------------------------------------------------------------------------------------------------------
def l1a(p, relu=1):
    L, lib = _lib()
    pa = L.L1AParams()
    _fill(pa.w, p["w"]); _fill(pa.root, p["root"]); _fill(pa.scale, p["scale"]); _fill(pa.shift, p["shift"])
    pa.relu = relu
    frag = (C.c_float * L.L1A_TC_WFRAG_FLOATS)()
    L.check(lib.dagr_l1a_tc_weights(C.byref(pa), C.cast(frag, C.c_void_p)), "l1a_tc_weights")
    return pa, torch.from_numpy(np.frombuffer(frag, np.float32).copy()).cuda()


def run_build(s, pa, wfrag, defer, tc=True, min_idx=0, xa0=None, cellmask0=None, flags=None):
    L, lib = _lib()
    N = s.N
    nbr = torch.zeros(16 * N, dtype=torch.int32, device="cuda")
    off = torch.zeros(16 * N, dtype=torch.int16, device="cuda")
    cellmask = (torch.zeros(s.cells, dtype=torch.int32) if cellmask0 is None else cellmask0.int()).cuda()
    xa = (torch.full((2 * N * 8,), NAN) if xa0 is None else xa0).cuda()
    wl_hdr = torch.zeros(2, dtype=torch.int32, device="cuda")
    wl_ids = torch.zeros(s.cells, dtype=torch.int32, device="cuda")
    head = (C.byref(s.geom.c_geom), N, P(s.start), P(s.ti), P(s.xyb), P(s.feat_s))
    tail = (P(flags), min_idx, P(nbr), P(off), P(cellmask), P(xa), P(wl_hdr), P(wl_ids), defer, st())
    if tc:
        L.check(lib.dagr_l1_build_tc(*head, C.byref(pa), P(wfrag), *tail), "l1_build_tc")
    else:
        L.check(lib.dagr_l1_build(*head, pa if pa is None else C.byref(pa), *tail), "l1_build")
    torch.cuda.synchronize()
    return dict(nbr=nbr.view(16, N).long().cpu(), off=(off.view(16, N).int() & 0xffff).long().cpu(), cellmask=cellmask.long().cpu() & 0xffffffff,
                xa=xa.cpu(), rows=xa_unpack(xa, N), beyond=int(wl_hdr[0]))


def l1b(p, relu=1, pool_mean=0):
    L, lib = _lib()
    pb = L.L1BParams()
    _fill(pb.w, p["w"]); _fill(pb.root, p["root"]); _fill(pb.skip, p["skip"][16:19])
    _fill(pb.scale, p["scale"]); _fill(pb.shift, p["shift"]); _fill(pb.sscale, p["sscale"]); _fill(pb.sshift, p["sshift"])
    pb.relu, pb.pool_mean = relu, pool_mean
    frag = (C.c_float * L.L1_TC_WFRAG_FLOATS)()
    w, root = np.ascontiguousarray(p["w"], np.float32), np.ascontiguousarray(p["root"], np.float32)
    L.check(lib.dagr_l1_tc_weights(w.ctypes.data, root.ctypes.data, 16, C.cast(frag, C.c_void_p)), "tc_weights")
    return pb, torch.from_numpy(np.frombuffer(frag, np.float32).copy()).cuda()


def run_conv_b(s, pb, wfrag, xa_flat, defer, skip_pre=None, x1=True, min_idx=0, persist0=None, ldx=24):
    L, lib = _lib()
    N, cells = s.N, s.cells
    x1b = torch.full((N, 16), NAN, device="cuda") if x1 else None
    persist = None if persist0 is None else persist0.clone().cuda()
    cnt = torch.full((cells,), -7, dtype=torch.int32, device="cuda")
    pxy = torch.full((cells, 2), -7, dtype=torch.int32, device="cuda")
    tmean, tmax = torch.full((cells,), NAN, device="cuda"), torch.full((cells,), NAN, device="cuda")
    xg = torch.full((cells, ldx), 7.0, device="cuda")
    wl_hdr = torch.zeros(2, dtype=torch.int32, device="cuda")
    wl_ids = torch.zeros(cells, dtype=torch.int32, device="cuda")
    xa_d, skip_d = xa_flat.cuda(), None if skip_pre is None else skip_pre.cuda()
    L.check(lib.dagr_l1_conv_b_pool_voxel_tc(C.byref(s.geom.c_geom), N, P(s.start), P(s.xyb), P(s.ti), P(s.feat_s),
                                             P(xa_d), P(s.nbr_d), P(s.off_d), C.byref(pb), P(wfrag),
                                             P(skip_d), min_idx, P(persist), P(x1b),
                                             P(cnt), P(pxy), P(tmean), P(tmax), P(xg), ldx, P(wl_hdr), P(wl_ids), defer, st()),
            "conv_b")
    torch.cuda.synchronize()
    c = lambda t: None if t is None else t.cpu()                                     # noqa: E731
    return dict(x1=c(x1b), persist=c(persist), cnt=cnt.cpu(), pxy=pxy.cpu(), tmean=tmean.cpu(), tmax=tmax.cpu(), xg=xg.cpu(),
                beyond=int(wl_hdr[0]))


def l1img(p):
    L, lib = _lib()
    pi = L.L1ImgParams()
    w = np.zeros((15, 24, 16), np.float32); w[:, :19] = p["w"]
    r = np.zeros((24, 16), np.float32); r[:19] = p["root"]
    k = np.zeros((24, 16), np.float32); k[:19] = p["skip"]
    _fill(pi.w, w); _fill(pi.root, r); _fill(pi.skip, k)
    _fill(pi.scale, p["scale"]); _fill(pi.shift, p["shift"]); _fill(pi.sscale, p["sscale"]); _fill(pi.sshift, p["sshift"])
    pi.relu = 1
    frag = (C.c_float * L.L1_TC_WFRAG_FLOATS)()
    L.check(lib.dagr_l1_tc_weights(w.ctypes.data, r.ctypes.data, 24, C.cast(frag, C.c_void_p)), "tc_weights")
    return pi, torch.from_numpy(np.frombuffer(frag, np.float32).copy()).cuda()


def run_image(s, pi, wfrag, x0_flat, xa_in, defer, inc=None, skip0=None):
    """dagr_l1_conv_a_image_tc (inc None) or _inc(min_idx = inc) on a copy of xa_in -> (xa rows, skipv)"""
    L, lib = _lib()
    N = s.N
    xa = xa_in.clone().cuda()
    skipv = (torch.full((N, 16), NAN) if skip0 is None else skip0.clone()).cuda()
    wl_hdr = torch.zeros(2, dtype=torch.int32, device="cuda")
    wl_ids = torch.zeros(s.cells, dtype=torch.int32, device="cuda")
    g = C.byref(s.geom.c_geom)
    x0_d = x0_flat.cuda()
    if inc is None:
        L.check(lib.dagr_l1_conv_a_image_tc(g, N, P(s.start), P(s.xyb), P(s.feat_s), P(x0_d), P(s.nbr_d), P(s.off_d),
                                            C.byref(pi), P(wfrag), P(xa), P(skipv), P(wl_hdr), P(wl_ids), defer, st()), "image")
    else:
        L.check(lib.dagr_l1_conv_a_image_inc(g, N, P(s.start), P(s.xyb), P(s.ti), P(s.feat_s), P(x0_d), P(s.nbr_d),
                                             P(s.off_d), C.byref(pi), P(wfrag), inc, P(xa), P(skipv), P(wl_hdr), P(wl_ids), defer,
                                             st()), "image_inc")
    torch.cuda.synchronize()
    return dict(xa=xa.cpu(), rows=xa_unpack(xa, N), skipv=skipv.cpu(), beyond=int(wl_hdr[0]))


# ------------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------------
CASES = {
    # the instance case: background, a 14000-event voxel (dense kernels' global / gathered paths), a 3000-event voxel
    # (dense staged, sparse neighbours over the conv capacity), a 1700-event voxel (lean launch over capacity)
    "640x480": dict(W=640, H=480, B=1, seed=3, n_bg=20000, clusters=[(0, 26, 16, 14000), (0, 8, 8, 3000), (0, 45, 30, 1700)],
                    border=500),
    "1280x720": dict(W=1280, H=720, B=1, seed=4, n_bg=30000, clusters=[(0, 20, 20, 2500)], border=500),
    "320x215_K8": dict(W=320, H=215, B=1, seed=5, n_bg=8000, K=8, clusters=[(0, 10, 10, 1500)], border=250),
    "240x180_B3": dict(W=240, H=180, B=3, seed=6, n_bg=6000, empty=(1,), border=250),
    "320x215_K1": dict(W=320, H=215, B=1, seed=7, n_bg=5000, K=1, border=250),
    "exact_512": dict(W=512, H=512, B=1, seed=8, n_bg=15000, radius=6.5 / 512, clusters=[(0, 20, 20, 2500)], border=250,
                      exact=True),
    "exact_1024": dict(W=1024, H=1024, B=1, seed=9, n_bg=8000, radius=14.5 / 1024, region=(256, 256), exact=True),
    # r = 13 on 23 x 25 px voxels: the dense build instance does not fit the shared memory, defer = 1 takes the lean launch
    "1280x960": dict(W=1280, H=960, B=1, seed=10, n_bg=30000, clusters=[(0, 20, 20, 2500)], border=500),
}
DENSE_BUILD_OVERFLOWS = ("exact_1024", "1280x960")


def dense_build_fits(geom):
    """whether dagr_l1_build[_tc] can run its dense instance at this geometry on this device (the launcher's own test)"""
    return build_dense_smem_bytes(geom) + 128 <= torch.cuda.get_device_properties(0).shared_memory_per_block_optin


@lru_cache(maxsize=None)
def stream(name):
    kw = dict(CASES[name])
    kw.pop("exact", None)
    s = Stream(**kw)
    # the adjacency every conv reads: the build kernel's, asserted equal to the oracle's in test_build
    pa, wf = l1a(build_params(np.random.default_rng(0), False))
    b = run_build(s, pa, wf, 0)
    s.nbr_d = b["nbr"].int().reshape(-1).cuda()
    s.off_d = b["off"].short().reshape(-1).cuda()
    return s


def exact(name):
    return bool(CASES[name].get("exact"))


def ref_build(s, p, relu=True):
    v, S = ref_conv(s.geom, s.ev3(), s.edges, s.pos[:, :2], p["w"], p["root"])
    sc, sh = torch.from_numpy(p["scale"]).double(), torch.from_numpy(p["shift"]).double()
    out, S = v * sc + sh, S * sc.abs() + sh.abs()
    return (out.clamp(min=0) if relu else out), S, v


def check(name, out, ref, S, c, ex):
    """exact tier: bit for bit; realistic: the per-element bound (c per node broadcast over channels)"""
    if ex:
        assert torch.equal(out, ref.float()), (name, float((out.double() - ref).abs().max()))
        return report(name, 0.0)
    r = report(name, bound_ratio(out, ref, S, c))
    assert r <= 1.0, (name, r)
    return r


# ------------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_build_against_float64_in_every_instance(name):
    s, ex = stream(name), exact(name)
    rng = np.random.default_rng(11)
    p = build_params(rng, ex, pol_zero=name == "exact_1024")
    pa, wf = l1a(p)
    nbr, off, deg, mask, _ = s.expected_adjacency()
    ref, S, _ = ref_build(s, p)
    c = (C_BUILD_TC + s.deg.double())[:, None]
    if ex:
        ax = s.ev3().abs()
        chans = (1, 2) if name == "exact_1024" else (0, 1, 2)                    # 1024: the polarity weights are zero
        amax = float(max(torch.bincount(s.edges[1], weights=ax[s.edges[0], k], minlength=s.N).max() for k in chans))
        a_step = 2.0 ** -(6 if s.geom.W == 512 else 8) * 2.0 ** -(9 if s.geom.W == 512 else 10)
        print("exact tier bits", exact_tier_budget(amax, a_step, S.numpy(), a_step * 2.0 ** -1 * 2.0 ** -1))
    runs = {}
    fits = dense_build_fits(s.geom)
    assert fits == (name not in DENSE_BUILD_OVERFLOWS), (name, build_dense_smem_bytes(s.geom))
    for defer in (0, 1):
        o = runs[defer] = run_build(s, pa, wf, defer)
        valid = nbr >= 0
        assert torch.equal(o["nbr"][valid], nbr[valid]) and torch.equal(o["off"][valid], off[valid]), (name, defer)
        assert torch.equal(o["nbr"][15], deg), (name, defer)
        assert torch.equal(o["cellmask"], mask), (name, defer)
        # defer = 1 where the dense instance does not fit: the lean launch, counting the voxels over its capacity
        cap = CAPS["BUILD"] if defer and fits else CAPS["BUILD_LEAN"]
        assert o["beyond"] == int(((s.nown > 0) & (s.total > cap)).sum()), (name, defer)
        check(f"build_tc/{name}/defer{defer}", s.sorted_to_arrival(o["rows"]), ref, S, c, ex)
    assert all(torch.equal(runs[0]["xa"], o["xa"]) for o in runs.values()), name
    # the fp32 form against the same reference (its own bound), and its adjacency-only form
    o = run_build(s, pa, None, 1, tc=False)
    if not ex:
        r = report(f"build_fp32/{name}", bound_ratio(s.sorted_to_arrival(o["rows"]), ref, S, (C_BUILD_FP32 + s.deg.double())[:, None]))
        assert r <= 1.0
    a = run_build(s, None, None, 0, tc=False)
    assert torch.equal(a["nbr"][nbr >= 0], nbr[nbr >= 0]) and torch.equal(a["cellmask"], mask)
    assert a["xa"].isnan().all(), "the adjacency-only form writes no activations"
    if name == "640x480":
        k = s.classes
        for cls in ("build_lean_staged", "build_lean_global", "build_staged", "build_dense_staged", "build_dense_global"):
            assert k[cls].sum() >= 3, (cls, int(k[cls].sum()))
    if name in ("320x215_K1", "640x480"):
        d = s.deg
        assert (d == 0).sum() > 0 and (name == "320x215_K1" or (d == 15).sum() > 1000), "degree 0 and full rows"


@pytest.mark.parametrize("name", ["640x480", "exact_512"])
def test_build_incremental_writes_only_new_nodes_and_ors_the_cellmask(name):
    s, ex = stream(name), exact(name)
    pa, wf = l1a(build_params(np.random.default_rng(12), ex))
    full = run_build(s, pa, wf, 1)
    m = s.N // 2
    prior = torch.from_numpy(np.random.default_rng(1).integers(0, 1 << 9, s.cells)).long() & ~16
    for defer in (0, 1):
        o = run_build(s, pa, wf, defer, min_idx=m, cellmask0=prior)
        new = s.perm >= m                                            # sorted positions of new nodes
        assert torch.equal(o["rows"][new], full["rows"][new]), (name, defer)
        assert o["rows"][~new].isnan().all(), "older nodes must not be written"
        assert torch.equal(o["cellmask"], prior | new_mask(s, m)), (name, defer)


def image_mode_build(s, p19):
    """the engine's first image step: dagr_l1_build_tc with the event-channel rows, scale 1 / shift 0 / no ReLU"""
    pe = dict(w=p19["w"][:, 16:19], root=p19["root"][16:19], scale=np.ones(16, np.float32), shift=np.zeros(16, np.float32))
    pa, wf = l1a(pe, relu=0)
    return pe, pa, wf


@pytest.mark.parametrize("name", ["640x480", "1280x720", "exact_512"])
def test_build_image_mode_gives_the_event_channel_partial_sums(name):
    s, ex = stream(name), exact(name)
    p19 = conv_params(np.random.default_rng(13), ex, cin=19)
    pe, pa, wf = image_mode_build(s, p19)
    v, S = ref_conv(s.geom, s.ev3(), s.edges, s.pos[:, :2], pe["w"], pe["root"])
    for defer in (0, 1):
        o = run_build(s, pa, wf, defer)
        check(f"build_image/{name}/defer{defer}", s.sorted_to_arrival(o["rows"]), v, S, (C_BUILD_TC + s.deg.double())[:, None], ex)


def ref_conv_b(s, p, X, skip_pre=None, relu=True):
    v, S = ref_conv(s.geom, X, s.edges, s.pos[:, :2], p["w"], p["root"])
    d = lambda k: torch.from_numpy(p[k]).double()                                  # noqa: E731
    y, Sy = v * d("scale") + d("shift"), S * d("scale").abs() + d("shift").abs()
    if skip_pre is None:
        e = s.ev3()
        sk = (e @ d("skip")[16:19]) * d("sscale") + d("sshift")
        Ss = (e.abs() @ d("skip")[16:19].abs()) * d("sscale").abs() + d("sshift").abs()
    else:
        sk = s.sorted_to_arrival(skip_pre).double()
        Ss = sk.abs()
    out = y + sk
    return (out.clamp(min=0) if relu else out), Sy + Ss


def check_pool(name, s, o, ref, S, c, ex, mean=False):
    """cnt, pxy, tmean, tmax exactly; xg per voxel against float64 max / mean of the node references"""
    cells, nown = s.cells, torch.from_numpy(s.nown)
    assert torch.equal(o["cnt"].long(), nown), name
    ne = nown > 0
    cl = s.cell_of
    T, W, H = s.geom.T, s.geom.W, s.geom.H
    st_ = torch.zeros(cells, dtype=torch.float64).index_add_(0, cl, s.pos[:, 2].double())
    sx = torch.zeros(cells, dtype=torch.float64).index_add_(0, cl, s.pos[:, 0].double())
    sy = torch.zeros(cells, dtype=torch.float64).index_add_(0, cl, s.pos[:, 1].double())
    tm = torch.full((cells,), -1.0, dtype=torch.float64).scatter_reduce(0, cl, s.pos[:, 2].double(), "amax")
    n = nown.double().clamp(min=1)
    want_tmean = torch.where(ne, (st_ / (n * T)).float(), torch.zeros(cells))
    want_tmax = torch.where(ne, (tm / T).float(), torch.zeros(cells))
    assert torch.equal(o["tmean"], want_tmean) and torch.equal(o["tmax"], want_tmax), name
    from oracle.ref_ops import round_to_pixel
    for k, (sv, size) in enumerate(((sx, W), (sy, H))):
        mean_f = (sv / (n * size)).float()                                      # the correctly rounded mean position
        inv = 1 / torch.tensor([float(size)])                                   # wh_inv of pooling.py:32
        assert (o["pxy"][~ne, k] == 0).all(), (name, k)
        assert torch.equal(o["pxy"][ne, k].float() * inv, round_to_pixel(mean_f, inv)[ne]), (name, k)
    assert (o["xg"][:, 16:] == 7.0).all(), "columns past 16 of a wider xg row must stay untouched"
    xg = o["xg"][:, :16].double()
    assert (xg[~ne] == 0).all(), name
    bnd = c * U * S + 2 * U * ref.abs()
    if mean:
        rv = torch.zeros(cells, 16, dtype=torch.float64).index_add_(0, cl, ref) / n[:, None]
        bv = torch.zeros(cells, 16, dtype=torch.float64).index_add_(0, cl, bnd + (nown[cl, None] + 1) * U * ref.abs()) / n[:, None]
    else:
        rv = torch.full((cells, 16), -np.inf, dtype=torch.float64).scatter_reduce(0, cl[:, None].expand(-1, 16), ref, "amax")
        bv = torch.zeros(cells, 16, dtype=torch.float64).scatter_reduce(0, cl[:, None].expand(-1, 16), bnd, "amax")
    if ex and not mean:
        assert torch.equal(xg[ne], rv[ne]), name
        return 0.0
    err = (xg - rv).abs()[ne]
    r = float(torch.where(err == 0, torch.zeros_like(err), err / bv[ne]).max())
    report(f"{name}/xg", r)
    assert r <= 1.0, (name, r)


@pytest.mark.parametrize("name", list(CASES))
def test_conv_b_against_float64_in_all_three_instances(name):
    s, ex = stream(name), exact(name)
    rng = np.random.default_rng(14)
    p = conv_params(rng, ex)
    X = node_rows(rng, s.N, ex, bits=3 if name == "exact_1024" else 4)        # node rows in sorted order
    xa = xa_pack(X)
    Xa = s.sorted_to_arrival(X)
    c = (C_CONV + s.deg.double())[:, None]
    ref, S = ref_conv_b(s, p, Xa)
    if ex:
        print("exact tier bits", exact_tier_budget(float(Xa.abs().max()) * 16, 2.0 ** -8, S.numpy(), 2.0 ** -13))
    pb, wf = l1b(p)
    pbm, _ = l1b(p, pool_mean=1)
    skip_pre = node_rows(rng, s.N, ex)
    pbg, _ = l1b(p, relu=0)
    refg, Sg = ref_conv_b(s, p, Xa, skip_pre=skip_pre, relu=False)
    out = {}
    for defer in (0, 1):
        plain = run_conv_b(s, pb, wf, xa, defer, x1=False)
        gen_relu = run_conv_b(s, pb, wf, xa, defer)                  # the general instance with the PLAIN arithmetic
        gen = run_conv_b(s, pbg, wf, xa, defer, skip_pre=skip_pre)
        mean = run_conv_b(s, pbm, wf, xa, defer)
        out[defer] = (plain, gen_relu, gen, mean)
        nb = int(((s.nown > 0) & (s.total > CAPS["CONV"])).sum())
        assert plain["beyond"] == gen["beyond"] == mean["beyond"] == nb, (name, defer)
        check(f"conv_b/{name}/defer{defer}/x1", s.sorted_to_arrival(gen_relu["x1"]), ref, S, c, ex)
        check(f"conv_b/{name}/defer{defer}/x1_skip_pre", s.sorted_to_arrival(gen["x1"]), refg, Sg, c, ex)
        for k in ("xg", "cnt", "pxy", "tmean", "tmax"):
            assert torch.equal(plain[k], gen_relu[k]), (name, defer, k)
        check_pool(f"conv_b/{name}/defer{defer}/max", s, plain, ref, S, c, ex)
        check_pool(f"conv_b/{name}/defer{defer}/max_skip_pre", s, gen, refg, Sg, c, ex)
        check_pool(f"conv_b/{name}/defer{defer}/mean", s, mean, ref, S, c, ex, mean=True)
        assert torch.equal(mean["x1"], gen_relu["x1"]), "pool_mean changes the pooling only"
    # node rows and max pooling are the same bits in every instance; the mean's per-voxel sum runs over another number of
    # warps in the dense kernel (include/dagr_b200.h says so), so it is held to its bound above and only its node rows are
    # compared here
    for i in range(4):
        for k, v in out[0][i].items():
            if k != "beyond" and not (i == 3 and k == "xg"):
                assert v is None or torch.equal(v, out[1][i][k]), (name, i, k)
    if name == "640x480":
        for cls in ("conv_staged", "conv_dense_staged", "conv_dense_gathered"):
            assert s.classes[cls].sum() >= 3, (cls, int(s.classes[cls].sum()))


@pytest.mark.parametrize("name", ["640x480", "exact_512"])
def test_conv_b_incremental_keeps_old_rows_and_folds_persist(name):
    s, ex = stream(name), exact(name)
    rng = np.random.default_rng(15)
    p = conv_params(rng, ex)
    X = node_rows(rng, s.N, ex)
    xa = xa_pack(X)
    pb, wf = l1b(p)
    full = run_conv_b(s, pb, wf, xa, 1)
    m = s.N // 2
    new = s.perm >= m
    persist0 = torch.from_numpy(rng.standard_normal((s.cells, 16)).astype(np.float32))
    for defer in (0, 1):
        o = run_conv_b(s, pb, wf, xa, defer, min_idx=m, persist0=persist0)
        assert torch.equal(o["x1"][new], full["x1"][new]), (name, defer)
        assert o["x1"][~new].isnan().all(), "older nodes' x1 rows must be untouched"
        sel = torch.nonzero(new).flatten()
        cl = s.cell_of[s.perm[sel]]
        mx = torch.full((s.cells, 16), -np.inf).scatter_reduce(0, cl[:, None].expand(-1, 16), full["x1"][sel], "amax")
        want = torch.maximum(mx, persist0)
        ne = torch.from_numpy(s.nown > 0)
        assert torch.equal(o["persist"][ne], want[ne]) and torch.equal(o["xg"][ne, :16], want[ne]), (name, defer)
        assert torch.equal(o["persist"][~ne], persist0[~ne]) and (o["xg"][~ne, :16] == 0).all()
        for k in ("cnt", "pxy", "tmean", "tmax"):
            assert torch.equal(o[k], full[k]), (name, k)


def ref_image(s, p, X0a, parta):
    """float64 BN(part + conv16(x0)) with ReLU, and skipv = BN_s(Linear over the 19 channels); arrival order"""
    v, S = ref_conv(s.geom, X0a, s.edges, s.pos[:, :2], p["w"][:, :16], p["root"][:16])
    d = lambda k: torch.from_numpy(p[k]).double()                                  # noqa: E731
    pa = parta.double()
    o = ((pa + v) * d("scale") + d("shift")).clamp(min=0)
    So = (pa.abs() + S) * d("scale").abs() + d("shift").abs()
    x19 = torch.cat([X0a.double(), s.ev3()], 1)
    sk = (x19 @ d("skip")) * d("sscale") + d("sshift")
    Ss = (x19.abs() @ d("skip").abs()) * d("sscale").abs() + d("sshift").abs()
    return o, So, sk, Ss


@pytest.mark.parametrize("name", ["640x480", "1280x720", "240x180_B3", "320x215_K1", "exact_512", "exact_1024"])
def test_image_conv_against_float64_and_the_same_bits_in_every_instance(name):
    s, ex = stream(name), exact(name)
    rng = np.random.default_rng(16)
    p = conv_params(rng, ex, cin=19)
    X0 = node_rows(rng, s.N, ex, bits=3)
    part = node_rows(rng, s.N, ex, bits=3)
    x0, xa_in = xa_pack(X0), xa_pack(part)
    pi, wf = l1img(p)
    ref, S, sk, Ss = ref_image(s, p, s.sorted_to_arrival(X0), s.sorted_to_arrival(part))
    if ex:
        # x0 and part on 2^-2, slot weights on 2^-6 (512) / 2^-8 (1024), weights on 2^-2, BN scales on 2^-1, x / W on 2^-9 /
        # 2^-10: the rows' sums lie on 2^-11 / 2^-13 and the skip branch's on 2^-12 / 2^-13
        a_step, g_row, g_skip = (2.0 ** -8, 2.0 ** -11, 2.0 ** -12) if s.geom.W == 512 else (2.0 ** -10, 2.0 ** -13, 2.0 ** -13)
        amax = float(torch.bincount(s.edges[1], weights=s.sorted_to_arrival(X0).abs().double().max(1).values[s.edges[0]],
                                    minlength=s.N).max())
        print("exact tier bits", exact_tier_budget(amax, a_step, S.numpy(), g_row), exact_tier_budget(1.0, 1.0, Ss.numpy(), g_skip))
    c = (C_CONV + s.deg.double())[:, None]
    runs = {}
    for defer in (0, 1):
        o = runs[defer] = run_image(s, pi, wf, x0, xa_in, defer)
        assert o["beyond"] == int(((s.nown > 0) & (s.total > CAPS["CONV"])).sum()), (name, defer)
        check(f"image/{name}/defer{defer}/xa", s.sorted_to_arrival(o["rows"]), ref, S, c, ex)
        check(f"image/{name}/defer{defer}/skipv", s.sorted_to_arrival(o["skipv"]), sk, Ss, C_SKIP, ex)
        inc = run_image(s, pi, wf, x0, xa_in, defer, inc=0)
        assert torch.equal(inc["xa"], o["xa"]) and torch.equal(inc["skipv"], o["skipv"]), "_inc(min_idx=0) == _tc"
    # every node's rows are the same bits with defer 0 and 1 -- including the sparse voxels (<= 32 nodes) next to dense ones
    if name == "640x480":
        for cls in ("image_sparse_staged", "image_sparse_dense_staged", "image_sparse_gathered"):
            assert s.classes[cls].sum() >= 3, (cls, int(s.classes[cls].sum()))
        vox = torch.from_numpy(s.classes["image_sparse_dense_staged"])[s.cell_of[s.perm]]
        assert torch.equal(runs[0]["rows"][vox], runs[1]["rows"][vox]), "sparse voxels next to a dense cluster"
    assert torch.equal(runs[0]["xa"], runs[1]["xa"]) and torch.equal(runs[0]["skipv"], runs[1]["skipv"]), name
    # incremental: older nodes' xa rows (final activations) and skipv rows are untouched
    m = s.N // 2
    new = s.perm >= m
    sentinel = part.clone()
    sentinel[~new] = 1234.5
    for defer in (0, 1):
        o = run_image(s, pi, wf, x0, xa_pack(sentinel), defer, inc=m)
        assert torch.equal(o["rows"][new], runs[0]["rows"][new]) and torch.equal(o["skipv"][new], runs[0]["skipv"][new])
        assert (o["rows"][~new] == 1234.5).all() and o["skipv"][~new].isnan().all(), (name, defer)


@pytest.mark.parametrize("name", ["640x480", "exact_512"])
def test_image_chain_build_then_conv_is_the_19_channel_conv(name):
    """the engine's sequence: dagr_l1_build_tc with the event-channel weights, then dagr_l1_conv_a_image_tc on its xa"""
    s, ex = stream(name), exact(name)
    rng = np.random.default_rng(17)
    p = conv_params(rng, ex, cin=19)
    X0 = node_rows(rng, s.N, ex, bits=2)
    if ex:
        # the event channels' partial sums lie on the fine grid of x / W (2^-15 at 512 x 512): integer weights there and
        # 2-bit image features keep the sum of the two parts within 24 bits of that grid
        p["w"][:, 16:19], p["root"][16:19] = dyadic(rng, (15, 3, 16), 2, 0), dyadic(rng, (3, 16), 2, 0)
    _, pa, wfa = image_mode_build(s, p)
    pi, wf = l1img(p)
    x19 = torch.cat([s.sorted_to_arrival(X0).double(), s.ev3()], 1)
    v, S = ref_conv(s.geom, x19, s.edges, s.pos[:, :2], p["w"], p["root"])
    d = lambda k: torch.from_numpy(p[k]).double()                                  # noqa: E731
    ref = (v * d("scale") + d("shift")).clamp(min=0)
    Sr = S * d("scale").abs() + d("shift").abs()
    if ex:
        ax = s.ev3().abs()
        amax = float(max(torch.bincount(s.edges[1], weights=ax[s.edges[0], k], minlength=s.N).max() for k in range(3)))
        print("exact tier bits", exact_tier_budget(amax, 2.0 ** -15, Sr.numpy(), 2.0 ** -16))
    for defer in (0, 1):
        b = run_build(s, pa, wfa, defer)
        o = run_image(s, pi, wf, xa_pack(X0), b["xa"], defer)
        check(f"image_chain/{name}/defer{defer}", s.sorted_to_arrival(o["rows"]), ref, Sr, (C_IMAGE + s.deg.double())[:, None], ex)


def test_a_sample_gets_the_same_bits_in_every_batch():
    """sample rows at B = 1 == the same events as sample 1 of B = 3 and sample 16 of B = 17 (compared through perm)"""
    W, H = 240, 180
    b1, p1 = make_events(W, H, 1, 5000, 21, border=250)
    f1 = torch.from_numpy(np.random.default_rng(21).choice([-1.0, 1.0], len(b1)).astype(np.float32))
    streams = {1: Stream(W, H, 1, 21, 0, events=(b1, p1), feat=f1)}
    for B, at in ((3, 1), (17, 16)):
        bo, po = make_events(W, H, B, 3000, 22 + B)
        lo, hi = bo < at, bo > at
        bb = torch.cat([bo[lo], torch.full_like(b1, at), bo[hi]])
        pp = torch.cat([po[lo], p1, po[hi]])
        ff = torch.cat([torch.ones(int(lo.sum())), f1, -torch.ones(int(hi.sum()))])
        streams[B] = Stream(W, H, B, 21, 0, events=(bb, pp), feat=ff)
    rng = np.random.default_rng(23)
    pa, wfa = l1a(build_params(rng, False))
    p = conv_params(rng, False)
    pb, wfb = l1b(p)
    p19 = conv_params(rng, False, cin=19)
    pi, wfi = l1img(p19)
    X = torch.from_numpy(rng.standard_normal((len(b1), 16)).astype(np.float32))          # arrival order of the sample
    got = {}
    for B, s in streams.items():
        off = int((s.batch < (0 if B == 1 else (1 if B == 3 else 16))).sum())
        arr = torch.arange(len(b1)) + off                                                  # the sample's arrival ids
        Xs = torch.randn(s.N, 16)
        Xs[s.pos_of[arr]] = X
        b = run_build(s, pa, wfa, 1)
        s.nbr_d, s.off_d = b["nbr"].int().reshape(-1).cuda(), b["off"].short().reshape(-1).cuda()
        cb = run_conv_b(s, pb, wfb, xa_pack(Xs), 1)
        im = run_image(s, pi, wfi, xa_pack(Xs), xa_pack(Xs), 0)
        sel = s.pos_of[arr]
        got[B] = (b["rows"][sel], cb["x1"][sel], im["rows"][sel], im["skipv"][sel])
    for B in (3, 17):
        for i in range(4):
            assert torch.equal(got[B][i], got[1][i]), (B, i)


def test_xa_permute_round_trips_rows_exactly():
    L, lib = _lib()
    s = stream("240x180_B3")
    N = s.N
    A = torch.randn(N, 16, device="cuda")
    srt = torch.full((2 * N * 8,), NAN, device="cuda")
    L.check(lib.dagr_xa_permute(N, P(s.perm_d), N, P(srt), P(A), 0, st()), "gather")
    back = torch.zeros(N, 16, device="cuda")
    L.check(lib.dagr_xa_permute(N, P(s.perm_d), 0, P(srt), P(back), 1, st()), "scatter")
    torch.cuda.synchronize()
    assert torch.equal(xa_unpack(srt, N), A.cpu()[s.perm]) and torch.equal(back, A)
    # partial: gather only rows < n_old, scatter only rows >= n_old
    m = N // 3
    srt2 = torch.full((2 * N * 8,), NAN, device="cuda")
    L.check(lib.dagr_xa_permute(N, P(s.perm_d), m, P(srt2), P(A), 0, st()), "gather")
    torch.cuda.synchronize()
    rows = xa_unpack(srt2, N)
    old = s.perm < m
    assert torch.equal(rows[old], A.cpu()[s.perm[old]]) and rows[~old].isnan().all()
