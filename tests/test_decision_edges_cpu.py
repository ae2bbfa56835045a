"""Decision edges of the post-process without a GPU.

The NMS cases that tests/test_decision_edges_gpu.py feeds to k_postprocess_nms are built here: box pairs whose IoU lies
within an ulp of the threshold (found by a seeded search that also emulates the FMA-contracted IoU exactly) and
suppression chains.  On them the oracle's NMS (oracle/ref_ops.py) must equal torchvision.ops.nms, which pins the
reference at exactly these edges.  Also the argument contract of dagr_postprocess_nms: every bad input is refused with
DAGR_E_ARG and a message before anything is launched, and B == 0 launches nothing.

Rows are built in the decoded (cx, cy, w, h, obj, cls...) domain; the decisions are reasoned on the fp32 corners the
post-process derives from them (x1 = cx - w / 2, x2 = w + x1).
"""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest
import torch

F32 = np.float32
E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below returns before a launch
THRESHOLDS = (0.65, 0.45)      # the model's nms_thre and one in another binade; both round down to fp32


def up(x, n=1):
    for _ in range(n):
        x = np.nextafter(F32(x), F32(np.inf))
    return F32(x)


def down(x, n=1):
    for _ in range(n):
        x = np.nextafter(F32(x), F32(-np.inf))
    return F32(x)


def corners(cx, cy, w, h):
    """fp32 (cx, cy, w, h) -> (x1, y1, x2, y2), op for op as postprocess_network_output (model/utils.py:63-64)"""
    cx, cy, w, h = F32(cx), F32(cy), F32(w), F32(h)
    x1, y1 = cx - w / F32(2), cy - h / F32(2)
    return np.array([x1, y1, w + x1, h + y1], dtype=F32)


def _round_f32(q: Fraction):
    """q rounded to the nearest fp32, ties to even (float() rounds to fp64 first, which can round twice)"""
    d = F32(float(q))
    lo, hi = (d, up(d)) if Fraction(float(d)) <= q else (down(d), d)
    el, eh = q - Fraction(float(lo)), Fraction(float(hi)) - q
    if el != eh:
        return lo if el < eh else hi
    return lo if int(lo.view(np.uint32)) % 2 == 0 else hi


def _inter_areas(a, b):
    iw = max(min(a[2], b[2]) - max(a[0], b[0]), F32(0))
    ih = max(min(a[3], b[3]) - max(a[1], b[1]), F32(0))
    return iw * ih, (a[2] - a[0]) * (a[3] - a[1])


def iou_rounded(a, b):
    """torchvision's CPU IoU of a (higher ranked) with b: every product, sum and the quotient rounded to fp32 on its own"""
    inter, sa = _inter_areas(a, b)
    sb = (b[2] - b[0]) * (b[3] - b[1])
    return inter / (sa + sb - inter)


def iou_fused(a, b):
    """the same IoU with sa + sb contracted to fma(dx_b, dy_b, sa), as nvcc compiles the plain C expression"""
    inter, sa = _inter_areas(a, b)
    s = _round_f32(Fraction(float(b[2] - b[0])) * Fraction(float(b[3] - b[1])) + Fraction(float(sa)))
    return inter / (s - inter)


def knife_edge_pairs(thr, seed):
    """Seeded search for decoded rows (A, B), A ranked first, whose rounded IoU is one ulp above fl(thr) ("above"), equal
    to it ("equal") or one ulp below ("below"), and pairs whose rounded and fused IoU fall on opposite sides of fl(thr)
    ("split+": rounded suppresses, fused keeps; "split-": the reverse).  B shares A's centre and height, so the IoU is
    about w_B / w_A; consecutive fp32 widths of B walk it across the threshold.  Returns [(tag, rowA, rowB)]."""
    t = F32(thr)
    rng = np.random.default_rng(seed)
    want = {"above": 1, "equal": 1, "below": 1, "split+": 2, "split-": 2}
    got = {k: [] for k in want}
    seen = set()                               # consecutive widths of B can give the same corners

    def add(tag, ra, rb, b):
        if len(got[tag]) < want[tag] and (tag, tuple(b)) not in seen:
            seen.add((tag, tuple(b)))
            got[tag].append((tag, ra, rb))

    for _ in range(2000):
        cx, cy = F32(rng.uniform(20, 300)), F32(rng.uniform(20, 300))
        wa, h = F32(rng.uniform(16, 200)), F32(rng.uniform(16, 200))
        ra = (cx, cy, wa, h)
        a = corners(*ra)
        wb = down(wa * t, 48)
        for _ in range(96):
            rb = (cx, cy, wb, h)
            b = corners(*rb)
            r = iou_rounded(a, b)
            tag = "above" if r == up(t) else "equal" if r == t else "below" if r == down(t) else None
            if tag:
                add(tag, ra, rb, b)
            if down(t, 2) <= r <= up(t, 2) and (r > t) != (iou_fused(a, b) > t):
                add("split+" if r > t else "split-", ra, rb, b)
            wb = up(wb)
        if all(len(got[k]) == want[k] for k in want):
            break
    assert all(len(got[k]) == want[k] for k in want), {k: len(v) for k, v in got.items()}
    return [c for k in want for c in got[k]]


def chain_rows(n, k, thr=0.65):
    """n candidates in k chains (chain c is a row of boxes at height 20 + 12 c; member m at cx = 20 + 1.5 m, 10 x 10 px):
    neighbours overlap with IoU 8.5 / 11.5 > thr, boxes two apart with IoU 7 / 13 < thr.  Rank r is member r // k of chain
    r % k, so with k > 1 every link jumps k ranks and many cross a 32-bit word of the suppression matrix.  Greedy NMS keeps
    the even members: i kills i + 1, which would have killed i + 2.  Returns (rows [n, 4] cx cy w h, scores [n] in rank
    order, the ranks NMS keeps)."""
    assert 7 / 13 < thr < 8.5 / 11.5
    r = np.arange(n)
    rows = np.stack([20 + 1.5 * (r // k), 20 + 12 * (r % k), np.full(n, 10.0), np.full(n, 10.0)], 1).astype(F32)
    scores = (F32(0.9) - r.astype(F32) * F32(2.0 ** -10)).astype(F32)
    return rows, scores, r[(r // k) % 2 == 0]


def _nms_pair(boxes, scores, thr):
    import torchvision
    from oracle import ref_ops as R
    b, s = torch.from_numpy(np.asarray(boxes, dtype=F32)), torch.from_numpy(np.asarray(scores, dtype=F32))
    return R.nms(b, s, thr), torchvision.ops.nms(b, s, thr)


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_oracle_nms_equals_torchvision_at_knife_edge_iou(thr):
    pytest.importorskip("torchvision")
    from oracle import ref_ops as R
    t = F32(thr)
    assert float(t) <= thr                     # torchvision compares with the double threshold: the same decisions
    cases = knife_edge_pairs(thr, seed=11)
    for tag, ra, rb in cases:
        a, b = corners(*ra), corners(*rb)
        r = iou_rounded(a, b)
        ref = R.box_iou_one_to_many(torch.from_numpy(a), torch.from_numpy(b)[None])[0]
        assert ref.item() == float(r), (tag, a, b)                                 # the emulation is the oracle's IoU
        mine, tv = _nms_pair(np.stack([a, b]), [0.9, 0.8], thr)
        assert torch.equal(mine, tv), (tag, a, b, mine, tv)
        assert len(tv) == (1 if r > t else 2), (tag, r)
        if tag.startswith("split"):
            assert (iou_fused(a, b) > t) != (r > t)


@pytest.mark.parametrize("n,k", [(33, 1), (65, 1), (256, 1), (65, 13), (256, 13)])
def test_oracle_nms_equals_torchvision_on_suppression_chains(n, k):
    pytest.importorskip("torchvision")
    rows, scores, keep = chain_rows(n, k)
    boxes = np.stack([corners(*row) for row in rows])
    perm = np.random.default_rng(n + k).permutation(n)                           # anchor order != rank order
    mine, tv = _nms_pair(boxes[perm], scores[perm], 0.65)
    assert torch.equal(mine, tv)
    assert np.array_equal(np.sort(perm[tv.numpy()]), keep)


def test_fused_emulation_rounds_like_hardware_fma():
    """_round_f32 against products that are exact in fp64 and sums that are not: fp64 would double-round these"""
    rng = np.random.default_rng(5)
    for _ in range(2000):
        x, y, z = (F32(v) for v in rng.uniform(1, 100, 3))
        q = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        f = _round_f32(q)
        assert abs(Fraction(float(f)) - q) <= abs(Fraction(float(up(f))) - q)
        assert abs(Fraction(float(f)) - q) <= abs(Fraction(float(down(f))) - q)
    half = Fraction(float(up(F32(1.0)))) / 2 + Fraction(1, 2)                     # exactly between 1 and 1 + ulp
    assert _round_f32(half) == F32(1.0) and _round_f32(half + Fraction(1, 2 ** 60)) == up(F32(1.0))


def _nms(lib, pred=BAD, B=2, A=175, nc=2, det=BAD, ndet=BAD):
    return lib.dagr_postprocess_nms(pred, B, A, nc, 0.001, 0.65, 640, 480, 1, det, ndet, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(pred=None), "null"),
    (dict(det=None), "null"),
    (dict(ndet=None), "null"),
    (dict(nc=0), "nc"),
    (dict(nc=-3), "nc"),
    (dict(A=0), "A must"),
    (dict(A=257), "A must"),
    (dict(B=-1), "B must"),
])
def test_postprocess_nms_rejects_bad_arguments(kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _nms(lib, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_postprocess_nms" in msg and needle in msg, msg


def test_postprocess_nms_with_no_images_launches_nothing():
    """B == 0 returns DAGR_OK before any launch (the pointers are never touched; without a device a launch would fail)"""
    from dagr_b200 import _lib
    assert _nms(_lib.load(), B=0) == 0
