"""The two kernels that turn floats into discrete decisions, checked exactly where the decision flips.

k_postprocess_nms against oracle.ref_ops.postprocess_network_output (stable descending sort, strict IoU > thr, the
obj * cls^2 confidence quirk): knife-edge IoUs within an ulp of nms_thre, including pairs on which an FMA-contracted IoU
decides the other way; confidence exactly at conf_thre and one ulp below; score and class ties; the class-offset trick;
the word boundaries of the suppression matrix; degenerate and inf/NaN boxes; batches, nc and filtering.  Every
comparison is exact: ndet, and det including its zero padding behind ndet.

round_to_pixel (pool2-4 finalize) against torch.div(m + 1e-5, 1 / size, rounding_mode="floor") on windows of consecutive
fp32 means around every pixel boundary, and the mean-pooled feature cast (float)(sum / n), in the same launch.

The C-ABI is called directly through _lib.load().
"""
import numpy as np
import pytest
import torch

from tests.test_decision_edges_cpu import (F32, THRESHOLDS, chain_rows, corners, down, iou_fused, iou_rounded,
                                           knife_edge_pairs, up)

pytestmark = pytest.mark.gpu

W, H = 640, 480
CONF = 0.001


def _row(cx, cy, w, h, obj, cls):
    return [float(cx), float(cy), float(w), float(h), float(obj)] + [float(c) for c in cls]


def _pred(images, nc, A=None):
    """images: list of row lists -> fp32 [B, A, 5 + nc]; missing rows are all zero (score 0, below any conf_thre > 0)"""
    A = A or max(len(rows) for rows in images)
    p = torch.zeros((len(images), A, 5 + nc), dtype=torch.float32)
    for b, rows in enumerate(images):
        if rows:
            p[b, :len(rows)] = torch.tensor(rows, dtype=torch.float32)
    return p


def run_nms(pred, conf=CONF, thr=0.65, width=W, height=H, filtering=True):
    from dagr_b200 import _lib
    lib = _lib.load()
    B, A, D = pred.shape
    p = pred.cuda().contiguous()
    det = torch.full((B, A, 6), 7.0, device="cuda")                 # sentinels: every element must be written
    ndet = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    _lib.check(lib.dagr_postprocess_nms(_lib.ptr(p), B, A, D - 5, conf, thr, width, height, 1 if filtering else 0,
                                        _lib.ptr(det), _lib.ptr(ndet), _lib.stream_ptr()), "dagr_postprocess_nms")
    torch.cuda.synchronize()
    return det.cpu(), ndet.cpu()


def expected(pred, conf=CONF, thr=0.65, width=W, height=H, filtering=True):
    from oracle import ref_ops as R
    B, A, D = pred.shape
    out = R.postprocess_network_output(pred.clone(), D - 5, conf, thr, height, width, filtering)
    det, ndet = torch.zeros((B, A, 6)), torch.zeros(B, dtype=torch.int32)
    for b, o in enumerate(out):
        k = len(o["scores"])
        det[b, :k, :4], det[b, :k, 4], det[b, :k, 5] = o["boxes"], o["scores"], o["labels"].float()
        ndet[b] = k
    return det, ndet


def check_nms(pred, what, **kw):
    det, ndet = run_nms(pred, **kw)
    want, wndet = expected(pred, **kw)
    assert torch.equal(ndet, wndet), f"{what}: ndet {ndet.tolist()} != oracle {wndet.tolist()}"
    if torch.isnan(want).any() or torch.isnan(det).any():
        torch.testing.assert_close(det, want, rtol=0, atol=0, equal_nan=True, msg=lambda m: f"{what}: {m}")
    else:
        bad = (det != want).any(-1).nonzero().tolist()
        assert not bad, f"{what}: det differs at [b, row] {bad[:8]}: {det[tuple(bad[0])].tolist()} != {want[tuple(bad[0])].tolist()}"
    return det, ndet


# ------------------------------------------------------------------------------------------------------------------------
# NMS
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("thr", THRESHOLDS)
def test_nms_knife_edge_iou(thr):
    """one image per pair (A scored 0.9, B 0.8): rounded IoU one ulp above fl(thr) suppresses B, equal and one ulp below
    keep it; on the split pairs an FMA-contracted sa + sb decides the other way from torchvision's rounding"""
    t = F32(thr)
    cases = knife_edge_pairs(thr, seed=11)
    images = [[_row(*ra, 0.9, [1.0]), _row(*rb, 0.8, [1.0])] for _, ra, rb in cases]
    pred = _pred(images, 1)
    det, ndet = run_nms(pred, thr=thr)
    want, wndet = expected(pred, thr=thr)
    for b, (tag, ra, rb) in enumerate(cases):
        a, bb = corners(*ra), corners(*rb)
        r, f = iou_rounded(a, bb), iou_fused(a, bb)
        assert int(wndet[b]) == (1 if r > t else 2)
        assert int(ndet[b]) == int(wndet[b]) and torch.equal(det[b], want[b]), (
            f"{tag} pair at nms_thre {thr}: boxes {a.tolist()} (0.9), {bb.tolist()} (0.8); torchvision IoU {float(r)!r}, "
            f"fused IoU {float(f)!r}; kernel kept {int(ndet[b])}, oracle / torchvision keep {int(wndet[b])}")


def test_nms_confidence_boundary():
    """score * cc == conf_thre exactly is kept, one ulp below is dropped; cc = 0.5 makes the products exact, the other rows
    come from a seeded search over consecutive fp32 objectness values"""
    rng = np.random.default_rng(3)
    for conf in (0.001, 0.2):
        ct = F32(conf)
        rows, keep = [(F32(4) * ct, F32(0.5)), (down(F32(4) * ct), F32(0.5))], []
        found = {}
        for _ in range(100):
            if len(found) == 2:
                break
            cc = F32(rng.uniform(0.5, 1.0))
            o = down(ct / (cc * cc), 16)
            for _ in range(32):
                v = (o * cc) * cc
                if v == ct and "eq" not in found:
                    found["eq"] = (o, cc)
                elif v == down(ct) and "lo" not in found:
                    found["lo"] = (o, cc)
                o = up(o)
        rows += [found["eq"], found["lo"]]
        img = []
        for i, (obj, cc) in enumerate(rows):
            v = (obj * cc) * cc
            assert v == ct or v == down(ct)
            keep.append(bool(v >= ct))
            img.append(_row(30 + 40 * i, 100, 20, 20, obj, [cc, cc * F32(0.5)]))   # disjoint boxes, class 0 is the max
        det, ndet = check_nms(_pred([img], 2), f"conf_thre {conf}", conf=conf)
        assert int(ndet[0]) == sum(keep) == 2


def test_nms_score_and_class_ties():
    """equal final scores rank by anchor index (the oracle's stable sort); equal class scores pick the first class"""
    img = [_row(0, 0, 0, 0, 0, [0.0, 0.0, 0.0])] * 16
    img[3] = _row(100, 100, 20, 20, 0.9, [1.0, 0.5, 0.5])         # tie with anchor 10, overlapping (IoU 0.9): 3 wins
    img[10] = _row(101, 100, 20, 20, 0.9, [1.0, 0.5, 0.5])
    img[7] = _row(300, 100, 20, 20, 0.5, [0.7, 0.7, 0.2])          # class tie 0 / 1 -> 0; three equal scores, disjoint:
    img[2] = _row(340, 100, 20, 20, 0.5, [0.2, 0.7, 0.7])          # class tie 1 / 2 -> 1; output in anchor order 2, 5, 7
    img[5] = _row(380, 100, 20, 20, 0.5, [0.7, 0.2, 0.7])          # class tie 0 / 2 -> 0
    det, ndet = check_nms(_pred([img], 3), "ties")
    assert int(ndet[0]) == 4
    assert det[0, 0, 0].item() == 90.0                             # anchor 3's box, not anchor 10's (x1 = 91)
    assert det[0, 1:4, 0].tolist() == [330.0, 370.0, 290.0] and det[0, 1:4, 5].tolist() == [1.0, 0.0, 0.0]


def test_nms_class_offset():
    """different classes are never suppressed unless boxes wider than max(W, H) + 1 meet across the class offset"""
    md1 = max(W, H) + 1
    img = [_row(100, 100, 40, 40, 0.9, [1.0, 0.0]), _row(101, 100, 40, 40, 0.8, [0.0, 1.0]),   # kept: other class
           _row(700, 700, 1400, 1400, 0.7, [1.0, 0.0]),                                       # class 0, 1400 px
           _row(700 - md1, 700 - md1, 1400, 1400, 0.6, [0.0, 1.0])]                           # class 1: == after offset
    det, ndet = check_nms(_pred([img], 2), "class offset")
    assert int(ndet[0]) == 3 and det[0, 2, 0].item() == 0.0


@pytest.mark.parametrize("k", [1, 13])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 63, 64, 65, 255, 256])
def test_nms_word_boundaries_and_chains(n, k):
    """n candidates among A = 256 anchors (the rest below conf_thre, interleaved): k suppression chains whose links cross
    32-bit words (i kills i + 1, so i + 2 survives), and an image where the rank-0 box suppresses victims in the last word
    while everything between survives"""
    rng = np.random.default_rng(100 * n + k)
    rows, scores, keep = chain_rows(n, k)
    slots = rng.permutation(256)[:n]
    chain = [_row(0, 0, 0, 0, 0, [0.0])] * 256
    for r in range(n):
        chain[slots[r]] = _row(*rows[r], scores[r], [1.0])
    victims = min(5, n - 1)
    last = [_row(0, 0, 0, 0, 0, [0.0])] * 256
    for r in range(n):
        if r == 0 or r >= n - victims:
            box = (500, 300, 40, 40) if r == 0 else (500 + 0.25 * (n - r), 300, 40, 40)
        else:
            box = (10 + 20 * (r % 20), 10 + 20 * (r // 20), 10, 10)      # disjoint 10 px boxes on a 20 px lattice
        last[slots[r]] = _row(*box, F32(0.9) - F32(r) * F32(2.0 ** -10), [1.0])
    det, ndet = check_nms(_pred([chain, last], 1), f"n = {n}, k = {k}")
    assert int(ndet[0]) == len(keep) and int(ndet[1]) == n - victims


def test_nms_dense_random_overlaps():
    """A = 256 random boxes piled on a small area, three classes, random scores: long data-dependent suppression patterns"""
    rng = np.random.default_rng(8)
    images = []
    for b in range(6):
        xy = rng.uniform(70, 90, (256, 2))
        wh = rng.uniform(20, 30, (256, 2))
        obj = rng.uniform(0, 1, 256) * (rng.uniform(0, 1, 256) > 0.1)
        cls = rng.uniform(0, 1, (256, 3))
        images.append([_row(*xy[i], *wh[i], obj[i], cls[i]) for i in range(256)])
    pred = _pred(images, 3)
    cc = pred[..., 5:].max(-1).values
    ncand = (pred[..., 4] * cc * cc >= CONF).sum(-1)
    for thr in THRESHOLDS:
        _, ndet = check_nms(pred, f"dense random, nms_thre {thr}", thr=thr)
        assert (ndet < ncand - 20).all()                        # plenty of suppression in every image


def test_nms_degenerate_and_extreme_rows():
    """zero-area boxes (IoU 0/0 is never above the threshold), identical boxes, and w / h = inf (exp overflow: corners -inf
    and NaN) or so large that the area overflows: same inf / NaN boxes and the same decisions as the oracle"""
    inf = float("inf")
    img = [_row(50, 50, 0, 0, 0.9, [1.0]), _row(50, 50, 0, 0, 0.8, [1.0]),          # two identical points
           _row(100, 50, 0, 10, 0.7, [1.0]), _row(100, 50, 20, 20, 0.6, [1.0]),     # zero-width line inside a box
           _row(200, 50, 20, 20, 0.5, [1.0]), _row(200, 50, 20, 20, 0.4, [1.0]),    # identical boxes: second suppressed
           _row(300, 50, inf, 20, 0.35, [1.0]), _row(300, 50, 20, inf, 0.3, [1.0]), # exp(reg) = inf
           _row(300, 50, 20, 20, 0.25, [1.0]),
           _row(400, 60, 3e38, 3e38, 0.2, [1.0]), _row(400, 60, 3e38, 3e38, 0.15, [1.0]),   # area overflows to inf
           _row(400, 60, 20, 20, 0.1, [1.0])]
    det, ndet = check_nms(_pred([img], 1), "degenerate")
    assert torch.isnan(det[0, :int(ndet[0]), :4]).any() and torch.isinf(det[0, :int(ndet[0]), :4]).any()


@pytest.mark.parametrize("nc", [1, 2, 100])
def test_nms_batch_nc_and_filtering(nc):
    """B = 5 images with different ndet (image 3 has every row below conf_thre); filtering = 0 returns all A rows in
    anchor order with ndet = A"""
    rng = np.random.default_rng(nc)
    images = []
    for b in range(5):
        A = 175
        xy, wh = rng.uniform(0, 300, (A, 2)), rng.uniform(5, 80, (A, 2))
        obj = rng.uniform(0, 1, A) * (rng.uniform(0, 1, A) < 0.2 * (b + 1))
        if b == 3:
            obj = rng.uniform(0, 0.9 * CONF, A)
        cls = rng.uniform(0.5, 1, (A, nc))
        images.append([_row(*xy[i], *wh[i], obj[i], cls[i]) for i in range(A)])
    pred = _pred(images, nc)
    _, ndet = check_nms(pred, f"nc = {nc}")
    assert int(ndet[3]) == 0 and len(set(ndet.tolist())) >= 4
    det, ndet = check_nms(pred, f"nc = {nc}, filtering = 0", filtering=False)
    assert (ndet == 175).all()


# ------------------------------------------------------------------------------------------------------------------------
# round_to_pixel and the mean cast (dagr_grid_pool_finalize)
# ------------------------------------------------------------------------------------------------------------------------
SIZES = [180, 215, 240, 320, 480, 640, 720, 1280, 4096]
HALF = 8                                                   # window: 2 * HALF + 1 consecutive fp32 values per boundary


def _boundary_windows(size):
    """for every pixel boundary k in [1, size): consecutive fp32 means around k * fl(1/size) - 1e-5"""
    inv = float(F32(1) / F32(size))
    c = (np.arange(1, size, dtype=np.float64) * inv - 1e-5).astype(np.float32)
    bits = c.view(np.int32)[:, None] + np.arange(-HALF, HALF + 1, dtype=np.int32)[None]
    return bits.view(np.float32).reshape(-1)


def _floor_ref(m, size):
    return torch.div(torch.from_numpy(m) + 1e-5, 1 / torch.Tensor([size]), rounding_mode="floor")


@pytest.mark.parametrize("i", range(len(SIZES)))
def test_round_to_pixel_at_every_boundary(i):
    from dagr_b200 import _lib
    lib = _lib.load()
    sw, sh = SIZES[i], SIZES[(i + 1) % len(SIZES)]               # W != H: a swapped x / y shows
    mx, my = _boundary_windows(sw), _boundary_windows(sh)
    cells = max(len(mx), len(my))
    mx = np.concatenate([mx, np.full(cells - len(mx), 0.5, np.float32)])
    my = np.concatenate([my, np.full(cells - len(my), 0.5, np.float32)])
    for m, size in ((mx, sw), (my, sh)):                        # the reference index flips inside every window
        q = _floor_ref(m, size)[: (size - 1) * (2 * HALF + 1)].view(size - 1, 2 * HALF + 1)
        assert (q[:, 0] == torch.arange(0, size - 1)).all() and (q[:, -1] == torch.arange(1, size)).all(), size
    rng = np.random.default_rng(i)
    n = np.array([1, 3, 7], np.int32)[np.arange(cells) % 3]
    C = 3
    possum = np.stack([mx.astype(np.float64) * n, my.astype(np.float64) * n, rng.uniform(0, 1, cells) * n], 1)
    accsum = rng.standard_normal((cells, C)) * 37.0 * n[:, None]
    gr = _lib.Grid(nx=cells, ny=1, B=1, W=sw, H=sh, posxr=None, posyr=None)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()                  # noqa: E731
    d_possum, d_accsum, d_pcnt = dev(possum), dev(accsum), dev(n)
    d_ptmax = torch.zeros(cells, dtype=torch.int32, device="cuda")
    pxy = torch.full((cells, 2), -1, dtype=torch.int32, device="cuda")
    tmean, tmax = torch.empty(cells, device="cuda"), torch.empty(cells, device="cuda")
    x = torch.empty((cells, C), device="cuda")
    _lib.check(lib.dagr_grid_pool_finalize(gr, C, 1, None, _lib.ptr(d_accsum), _lib.ptr(d_possum), _lib.ptr(d_ptmax),
                                           _lib.ptr(d_pcnt), _lib.ptr(pxy), _lib.ptr(tmean), _lib.ptr(tmax), _lib.ptr(x),
                                           _lib.stream_ptr()), "dagr_grid_pool_finalize")
    torch.cuda.synchronize()
    n64 = torch.from_numpy(n).double()
    mean = (torch.from_numpy(possum) / n64[:, None]).float()
    assert torch.equal(mean[:, 0], torch.from_numpy(mx)) and torch.equal(mean[:, 1], torch.from_numpy(my))
    for col, m, size in ((0, mx, sw), (1, my, sh)):
        want = _floor_ref(m, size).long()
        got = pxy[:, col].cpu().long()
        bad = (got != want).nonzero().flatten()
        assert len(bad) == 0, (f"{'xy'[col]} at size {size}: {len(bad)} cells, first mean {m[bad[0]]!r}: "
                               f"{int(got[bad[0]])} != {int(want[bad[0]])}")
    assert torch.equal(tmean.cpu(), mean[:, 2])
    assert torch.equal(x.cpu(), (torch.from_numpy(accsum) / n64[:, None]).float())
