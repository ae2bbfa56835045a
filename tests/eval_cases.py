"""Seeded evaluation sets that reach the internal switches of csrc/evaluate.cu, for tests/test_eval_kernels_gpu.py (and pinned
without a GPU by tests/test_eval_cpu.py).  Each builder returns (gts, dts, K) in the DetectionBuffer layout: per image a dict
of float32 boxes [x1, y1, x2, y2] and int64 labels, with float32 scores for the detections."""
import numpy as np
import torch

EV_MAXDET = 100
RS_TILE = 2048                 # radix sort items per CTA (evaluate.cu)
AC_TILE = 2048                 # accumulation items per CTA (evaluate.cu)
EV_IOU_CAP = 800               # fp64 IoU entries a match warp stages
SCAN_CHUNK = 256 * 2048        # k_scan_blocksums carries across chunks of 256 block sums of 2048 counts


def _img(gb, gl, db, ds, dl):
    f = lambda v: torch.as_tensor(np.asarray(v, np.float32).reshape(-1, 4))
    return (dict(boxes=f(gb), labels=torch.as_tensor(np.asarray(gl, np.int64))),
            dict(boxes=f(db), scores=torch.as_tensor(np.asarray(ds, np.float32)), labels=torch.as_tensor(np.asarray(dl, np.int64))))


def _near(rng, g, n, jitter):
    """n detections around GT boxes g (rows picked at random), each corner moved by up to `jitter` pixels"""
    src = rng.integers(0, len(g), n)
    return g[src] + rng.uniform(-jitter, jitter, (n, 4)).astype(np.float32)


def _boxes(rng, n, span=600.0, lo=8.0, hi=120.0):
    xy = rng.uniform(0, span, (n, 2))
    wh = rng.uniform(lo, hi, (n, 2))
    return np.concatenate([xy, xy + wh], 1).astype(np.float32)


def kept_total(gts, dts, K):
    """detections the evaluator keeps: per image with GT and class in [0, K), the first 100 by score"""
    tot = 0
    for g, d in zip(gts, dts):
        if len(g["boxes"]) == 0:
            continue
        lab = d["labels"].numpy()
        for c in range(K):
            tot += min(int((lab == c).sum()), EV_MAXDET)
    return tot


def class_counts(gts, dts, K):
    """kept detections per class over the images with GT"""
    out = np.zeros(K, np.int64)
    for g, d in zip(gts, dts):
        if len(g["boxes"]):
            lab = d["labels"].numpy()
            for c in range(K):
                out[c] += min(int((lab == c).sum()), EV_MAXDET)
    return out


# ---- radix sort -----------------------------------------------------------------------------------------------------
def many_classes(K, seed, classes=None):
    """K classes, detections and GTs only in `classes` (default: every class >= 256, or the top 44 when K <= 256); with
    classes c and c + 256 both present the sort's ninth class bit decides their order"""
    rng = np.random.default_rng(seed)
    classes = list(classes) if classes is not None else (list(range(256, K)) if K > 256 else list(range(K - 44, K)))
    gts, dts = [], []
    for i in range(12):
        ng = int(rng.integers(2, 9))
        gb, gl = _boxes(rng, ng), rng.choice(classes, ng)
        nd = int(rng.integers(4, 30))
        src = rng.integers(0, ng, nd)
        db = gb[src] + rng.uniform(-10, 10, (nd, 4)).astype(np.float32)
        dl = np.where(rng.random(nd) < 0.15, rng.choice(classes, nd), gl[src])
        ds = np.round(rng.random(nd) * 20) / 20
        g, d = _img(gb, gl, db, ds, dl)
        gts.append(g)
        dts.append(d)
    return gts, dts, K


def kept_exactly(total, seed, K=2, equal_scores=False):
    """`total` kept detections over 2 classes and n images, plus detections that are dropped (beyond 100 per image and
    class, in images without GT, labels outside [0, K)); scores on a coarse grid (ties across tiles) or all equal"""
    rng = np.random.default_rng(seed)
    per = []                                                   # kept count per (image, class), <= 100
    left = total
    while left > 0:
        k = int(min(left, rng.integers(1, EV_MAXDET + 1)))
        per.append(k)
        left -= k
    gts, dts = [], []
    for j, k in enumerate(per):
        c = j % K
        ng = int(rng.integers(1, 7))
        gb = _boxes(rng, ng)
        gl = np.full(ng, c)
        gl[0] = (c + 1) % K                                    # one GT of the other class
        extra = 15 if j % 5 == 0 and k == EV_MAXDET else 0     # dropped: past the 100 cap
        n = k + extra
        db = _near(rng, gb, n, 12.0)
        ds = np.full(n, 0.5, np.float32) if equal_scores else (np.round(rng.random(n) * 16) / 16).astype(np.float32)
        dl = np.full(n, c)
        foreign = rng.integers(0, 3)
        db = np.concatenate([db, _boxes(rng, foreign)])
        ds = np.concatenate([ds, np.full(foreign, 0.5 if equal_scores else 0.9, np.float32)])
        dl = np.concatenate([dl, np.full(foreign, K + 3)])       # never kept
        g, d = _img(gb, gl, db, ds, dl)
        gts.append(g)
        dts.append(d)
        if j % 7 == 3:                                         # an image without GT: its detections are never kept
            g, d = _img(np.zeros((0, 4)), [], _boxes(rng, 4), [0.5 if equal_scores else 0.7] * 4, [c] * 4)
            gts.append(g)
            dts.append(d)
    return gts, dts, K


# ---- count scan ---------------------------------------------------------------------------------------------------------
def wide_scan(n_images=5300, K=100, seed=3):
    """n_images * K past one 256-chunk of scan block sums: one GT and up to two detections per image, classes spread over
    all K so keys land on both sides of the carry"""
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for i in range(n_images):
        gb = _boxes(rng, 1)
        c = int(rng.integers(0, K))
        nd = int(rng.integers(0, 3))
        db = _near(rng, gb, nd, 20.0)
        dl = np.where(rng.random(nd) < 0.3, rng.integers(0, K, nd), c)
        g, d = _img(gb, [c], db, (np.round(rng.random(nd) * 10) / 10).astype(np.float32), dl)
        gts.append(g)
        dts.append(d)
    return gts, dts, K


# ---- score keys ---------------------------------------------------------------------------------------------------------
def score_keys():
    """one GT per image; detections that all overlap it, ordered only by their score keys: -0.0 before +0.0 in the input
    (equal keys: input order decides), +-inf, NaN (last, as numpy sorts it), denormals and negative scores.  The box that
    comes first in the oracle's order has the higher IoU, so any reordering changes true / false positives."""
    f32 = np.float32
    den = np.array([1, 2, 0x7FFFFF], np.uint32).view(np.float32)          # smallest, next, largest denormal
    sets = [
        [-0.0, 0.0],
        [0.0, -0.0, 0.0],
        [-0.0, f32(den[0]), 0.0],
        [f32(den[1]), f32(den[0]), f32(den[2]), 0.0, -f32(den[0])],
        [np.inf, 1.0, -np.inf, np.nan, 0.5],
        [np.nan, -0.25, np.nan, -np.inf, -0.0],
        [-1.5, -0.5, -1e-30, -3e38, -1.5],
        [np.float32(np.finfo(np.float32).max), np.inf, np.finfo(np.float32).tiny, 0.0],
    ]
    gts, dts = [], []
    for j, s in enumerate(sets):
        gb = np.array([[100.0, 100.0, 200.0, 180.0]], np.float32)
        # detection k shifted right by 4k + 1 pixels: lower IoU the later it comes in input order
        db = np.array([[100.0 + 4 * k + 1, 100.0, 200.0 + 4 * k + 1, 180.0] for k in range(len(s))], np.float32)
        g, d = _img(gb, [j % 2], db, np.array(s, np.float32), [j % 2] * len(s))
        gts.append(g)
        dts.append(d)
        # the same scores across images: the accumulation's stable sort keeps image order
        g, d = _img(gb + 300, [j % 2], db[::-1] + 300, np.array(s, np.float32), [j % 2] * len(s))
        gts.append(g)
        dts.append(d)
    return gts, dts, 2


# ---- matcher --------------------------------------------------------------------------------------------------------------
def matcher(ng, nk, seed):
    """one image, ng GTs of class 0 (a few outside some area ranges) interleaved with class-1 GTs, nk detections of class 0
    near them: kept * ng decides the staged (fast) or recomputed (slow) path"""
    rng = np.random.default_rng(seed)
    gb0 = _boxes(rng, ng, span=900.0, lo=6.0, hi=140.0)
    gb1 = _boxes(rng, 5)
    gb = np.concatenate([gb0, gb1])
    gl = np.array([0] * ng + [1] * 5)
    perm = rng.permutation(len(gb))
    gb, gl = gb[perm], gl[perm]
    db = _near(rng, gb0, nk, 6.0)
    ds = (np.round(rng.random(nk) * 30) / 30).astype(np.float32)
    g, d = _img(gb, gl, db, ds, [0] * nk)
    return [g], [d], 2


def rank_ties(seed=11):
    """classes with more than 100 detections in one image whose scores tie across rank 99 / 100 / 101 (the first 100 in the
    stable order are kept), and a class with exactly 100"""
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for n, tie in ((100, (97, 103)), (101, (99, 101)), (102, (98, 102)), (140, (95, 130)), (130, (100, 102))):
        gb = _boxes(rng, 12)
        db = _near(rng, gb, n, 10.0)
        ds = np.sort((np.round(rng.random(n) * 1000) / 1000).astype(np.float32))[::-1].copy()
        ds[tie[0]:tie[1]] = ds[tie[0]]
        p = rng.permutation(n)                                   # input order is not score order
        g, d = _img(gb, [0] * 12, db[p], ds[p], [0] * n)
        gts.append(g)
        dts.append(d)
    return gts, dts, 1


def area_interleaved(seed=5):
    """GTs of the class interleaved with other classes and with GTs outside the small / medium / large ranges, detections
    that overlap both an in-range and an out-of-range GT: pass 0 (in range) must win over pass 1 (ignored) in input order"""
    rng = np.random.default_rng(seed)
    gts, dts = [], []
    for i in range(40):
        base = rng.uniform(0, 500, 2).astype(np.float32)
        sizes = [20.0, 31.5, 32.0, 40.0, 95.0, 96.0, 97.0, 150.0]
        gb, gl = [], []
        for k, s in enumerate(rng.permutation(sizes)):
            o = base + rng.uniform(-4, 4, 2).astype(np.float32)
            gb.append([o[0], o[1], o[0] + s, o[1] + s * float(rng.uniform(0.8, 1.2))])
            gl.append(0 if k % 3 else int(rng.integers(0, 3)))
        gb = np.array(gb, np.float32)
        nd = 12
        db = _near(rng, gb, nd, 5.0)
        dl = np.where(rng.random(nd) < 0.8, 0, rng.integers(0, 3, nd))
        g, d = _img(gb, gl, db, (np.round(rng.random(nd) * 8) / 8).astype(np.float32), dl)
        gts.append(g)
        dts.append(d)
    return gts, dts, 3


def slow_path_thresholds(seed=7):
    """more than 32 GTs of the class (the slow path, matched set in one gtm word per GT): detections placed so that a GT
    is the best match at low IoU thresholds and not at high ones, so several of its 40 (area, threshold) bits are set by
    different lanes"""
    rng = np.random.default_rng(seed)
    gb = np.array([[60.0 * (k % 8), 60.0 * (k // 8), 60.0 * (k % 8) + 50, 60.0 * (k // 8) + 50] for k in range(40)], np.float32)
    db, ds = [], []
    for k in range(0, 40, 2):
        x, y = gb[k, 0], gb[k, 1]
        db.append([x + 2, y, x + 52, y + 50])                  # IoU 48/52 ~ 0.92 with GT k
        db.append([x + 9, y, x + 59, y + 50])                  # IoU 41/59 ~ 0.69 with GT k, and 0 with GT k + 1 (gap of 10)
        db.append([x + 15, y + 3, x + 65, y + 53])
        ds += [0.9 - 0.01 * k, 0.95 - 0.01 * k, 0.6]
    g, d = _img(gb, [0] * 40, np.array(db, np.float32), np.array(ds, np.float32), [0] * len(ds))
    return [g], [d], 1


# ---- accumulation -------------------------------------------------------------------------------------------------------
def acc_tiles(seed=13):
    """classes holding AC_TILE - 1, AC_TILE and AC_TILE + 1 kept detections (their true positives run across the tile
    boundary, so recall buckets straddle it); a class whose first tile is all true positives (a detection equal to each GT,
    at the top score) and whose second tile is all false positives; a class with GT but no detection, one with detections
    but no GT, and the last class empty"""
    rng = np.random.default_rng(seed)
    K = 7
    gts, dts = [], []

    def add(gb, gl, db, ds, c):
        gb4 = _boxes(rng, 2, span=2000.0) + 20000                # class 4: GT only, never detected
        g, d = _img(np.concatenate([gb, gb4]), list(gl) + [4, 4], db, ds, [c] * len(db))
        gts.append(g)
        dts.append(d)

    for c, n in ((0, AC_TILE - 1), (1, AC_TILE), (2, AC_TILE + 1)):
        left = n
        while left > 0:
            k = min(left, EV_MAXDET)
            gb = _boxes(rng, 40, span=2000.0)
            add(gb, [c] * 40, _near(rng, gb, k, 15.0), (np.round(rng.random(k) * 64) / 64 * 0.9).astype(np.float32), c)
            left -= k
    left = AC_TILE                                               # class 3: AC_TILE true positives at 0.99
    while left > 0:
        k = min(left, 50)
        gb = _boxes(rng, 50, span=2000.0)
        add(gb, [3] * 50, gb[:k], np.full(k, 0.99, np.float32), 3)
        left -= k
    left = AC_TILE + 5                                           # then AC_TILE + 5 false positives at 0.98
    while left > 0:
        k = min(left, EV_MAXDET)
        add(_boxes(rng, 4, span=2000.0), [3] * 4, _boxes(rng, k, span=2000.0) + 10000, np.full(k, 0.98, np.float32), 3)
        left -= k
    add(_boxes(rng, 2), [0, 1], _boxes(rng, 30) + 3000, rng.random(30).astype(np.float32), 5)   # class 5: no GT
    return gts, dts, K


CASES = {
    "radix_k255": lambda: many_classes(255, 1),
    "radix_k256": lambda: many_classes(256, 2),
    "radix_k257": lambda: many_classes(257, 3),
    "radix_k300": lambda: many_classes(300, 4),
    "radix_k257_bit8": lambda: many_classes(257, 5, classes=(0, 1, 256)),
    "radix_k300_bit8": lambda: many_classes(300, 6, classes=(0, 43, 256, 299, 287)),
    "kept_2047": lambda: kept_exactly(2047, 1),
    "kept_2048": lambda: kept_exactly(2048, 2),
    "kept_2049": lambda: kept_exactly(2049, 3),
    "kept_4097": lambda: kept_exactly(4097, 4),
    "equal_scores_many_tiles": lambda: kept_exactly(5 * RS_TILE + 17, 5, K=1, equal_scores=True),
    "score_keys": score_keys,
    "match_ng32_nk25": lambda: matcher(32, 25, 1),
    "match_ng32_nk26": lambda: matcher(32, 26, 2),
    "match_ng33_nk10": lambda: matcher(33, 10, 3),
    "match_ng8_nk100": lambda: matcher(8, 100, 4),
    "match_ng9_nk89": lambda: matcher(9, 89, 5),
    "rank_ties": rank_ties,
    "area_interleaved": area_interleaved,
    "slow_path_thresholds": slow_path_thresholds,
    "acc_tiles": acc_tiles,
}
