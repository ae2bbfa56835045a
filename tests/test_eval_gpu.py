"""COCO bbox evaluation on the device (dagr_evaluate_bbox through dagr_b200.evaluation) against the restated COCOeval of
oracle/ref_coco.py: precision f64[10, 101, K, 4] and recall f64[10, K, 4] bit for bit, and the six summary stats equal."""
import numpy as np
import pytest
import torch

from dagr_b200 import evaluation
from oracle import ref_coco
from tests.helpers import make_inputs, make_model
from tests.test_eval_cpu import d, g, golden_case, GOLDEN

pytestmark = pytest.mark.gpu


def check(gts, dts, K):
    out = evaluation.accumulate(gts, dts, K)
    ev = ref_coco.evaluate_lists(gts, dts, K)
    if ev is None:
        assert out is None
        return None
    prec, rec = (t.cpu().numpy() for t in out)
    for name, got, want in (("precision", prec, ev.eval["precision"][..., 2]), ("recall", rec, ev.eval["recall"][..., 2])):
        bad = np.argwhere(got.view(np.int64) != want.view(np.int64))
        assert len(bad) == 0, f"{name}: {len(bad)} entries differ, first {bad[:3].tolist()}: " \
                              f"{[(got[tuple(b)], want[tuple(b)]) for b in bad[:3]]}"
    s = evaluation.summarize(prec)
    assert [s[k] for k in evaluation.OUT_KEYS] == ev.stats[:6].tolist()
    return ev


def cuda(dicts):
    return [{k: v.cuda() for k, v in x.items()} for x in dicts]


@pytest.mark.parametrize("name", ["k2", "k5", "nodet", "nogt"])
def test_golden_inputs_through_detection_buffer(name):
    gts, dets, K = golden_case(name)
    check(gts, dets, K)
    buf = evaluation.DetectionBuffer(480, 640, [f"c{k}" for k in range(K)])
    half = len(dets) // 2
    buf.update(dets[:half], gts[:half], "dsec")
    buf.update(cuda(dets[half:]), cuda(gts[half:]), "dsec")
    res = buf.compute()
    assert sorted(res) == [str(k) for k in GOLDEN[f"{name}_keys"]]
    assert [res[k] for k in sorted(res)] == GOLDEN[f"{name}_stats"].tolist()
    assert buf.detections == [] and buf.ground_truth == []


def _iou_family():
    """GT [0, 0, W, H], detection [s, 0, W + s, H] on a grid of float32-exact sizes and shifts, with the oracle's IoU"""
    W = np.arange(1, 401, dtype=np.float64)[:, None, None]
    H = np.array([1.0, 3.0, 7.0, 10.0, 13.0])[None, :, None]
    s = (np.arange(0, 801, dtype=np.float64) / 4)[None, None, :]
    w = np.minimum(W + s, W) - np.maximum(s, 0.0)
    i = w * H
    iou = i / ((W * H + W * H) - i)
    return np.broadcast_arrays(W, H, s, np.where(w > 0, iou, 0.0))


def test_iou_exactly_at_each_threshold_and_either_side():
    W, H, s, iou = _iou_family()
    gts, dts = [], []
    for t in evaluation.IOU_THRS:
        below, above = np.where(iou < t, iou, -1).max(), np.where(iou > t, iou, 2).min()
        for target in (t, below, above):
            hit = np.argwhere(iou == target)
            if len(hit) == 0:
                continue
            w, h, sh = (float(a[tuple(hit[0])]) for a in (W, H, s))
            gts.append(g([[0, 0, w, h]], [0]))
            dts.append(d([[sh, 0, w + sh, h]], [.5], [0]))
    assert len(gts) >= 25
    check(gts, dts, 1)


def test_areas_at_the_range_edges():
    f32 = np.float32
    gts, dts = [], []
    for side in (32, 96):
        for h in (np.nextafter(f32(side), f32(0)), f32(side), np.nextafter(f32(side), f32(200))):
            b = [0.0, 0.0, float(side), float(h)]
            gts.append(g([b, [5.0, 5.0, 5.0 + float(side), 5.0 + float(h)]], [0, 1]))
            dts.append(d([b, [5.0, 5.0, 5.0 + float(side), 5.0 + float(h)], [1.0, 1.0, 1.0 + float(side), float(h)]],
                         [.9, .8, .7], [0, 1, 0]))
    ev = check(gts, dts, 2)
    assert ev is not None


def test_score_ties_within_and_across_images():
    gts = [g([[0, 0, 50, 50], [60, 60, 120, 120]], [0, 0]) for _ in range(4)]
    dts = [d([[0, 0, 50, 50], [200, 200, 250, 250], [60, 60, 120, 120], [1, 1, 50, 50]], [.5, .5, .5, -0.0], [0, 0, 0, 0]),
           d([[300, 300, 350, 350], [60, 60, 120, 120]], [.5, .5], [0, 0]),
           d([[0, 0, 50, 50], [0, 0, 49, 50]], [0.0, .5], [0, 0]),
           d([[61, 60, 120, 120], [0, 0, 50, 50]], [.25, .25], [0, 0])]
    check(gts, dts, 1)


def test_more_than_100_detections_and_crowded_images():
    gen = torch.Generator().manual_seed(5)

    def rand_boxes(n, lo=0, span=300):
        xy = torch.rand(n, 2, generator=gen) * span + lo
        return torch.cat([xy, xy + torch.rand(n, 2, generator=gen) * 60 + 4], 1)

    gts, dts = [], []
    # 250 detections of one class (the first 100 by score are kept), few GTs: fast path
    gb = rand_boxes(6)
    gts.append(dict(boxes=gb, labels=torch.zeros(6, dtype=torch.long)))
    db = torch.cat([gb.repeat(40, 1) + torch.randn(240, 4, generator=gen) * 3, rand_boxes(10)])
    dts.append(dict(boxes=db, scores=torch.round(torch.rand(250, generator=gen) * 50) / 50, labels=torch.zeros(250, dtype=torch.long)))
    # 300 GTs of one class in one image (more than the 32 a warp stages), 150 detections near them
    gb = rand_boxes(300, span=800)
    gts.append(dict(boxes=gb, labels=torch.zeros(300, dtype=torch.long)))
    db = gb[torch.randint(0, 300, (150,), generator=gen)] + torch.randn(150, 4, generator=gen) * 4
    dts.append(dict(boxes=db, scores=torch.rand(150, generator=gen), labels=torch.zeros(150, dtype=torch.long)))
    # 20 GTs and 100 detections: within 32 GTs, but more IoU entries than a warp stages
    gb = rand_boxes(20)
    gts.append(dict(boxes=gb, labels=torch.zeros(20, dtype=torch.long)))
    db = gb.repeat(5, 1) + torch.randn(100, 4, generator=gen) * 5
    dts.append(dict(boxes=db, scores=torch.rand(100, generator=gen), labels=torch.zeros(100, dtype=torch.long)))
    # 33 GTs: just past the staged count, class 1 beside them on the fast path
    gb = rand_boxes(40)
    lab = torch.tensor([0] * 33 + [1] * 7)
    gts.append(dict(boxes=gb, labels=lab))
    dts.append(dict(boxes=gb + 1.5, scores=torch.rand(40, generator=gen), labels=lab.clone()))
    check(gts, dts, 2)


def test_images_without_gt_gt_without_detections_zero_width_and_foreign_labels():
    gts = [g([], []), g([[0, 0, 40, 40]], [1]), g([[10, 10, 10, 50], [0, 0, 30, 30]], [0, 0]),
           g([[0, 0, 20, 20], [5, 5, 25, 25]], [7, -1]), g([[0, 0, 64, 64]], [0])]
    dts = [d([[0, 0, 40, 40]], [.9], [0]), d([], [], []), d([[10, 10, 10, 50], [0, 0, 30, 30], [0, 0, 0, 0]], [.8, .7, .6], [0, 0, 0]),
           d([[0, 0, 20, 20], [5, 5, 25, 25], [0, 0, 64, 64]], [.9, .8, .7], [7, -1, 2 ** 32 + 1]),
           d([[0, 0, 64, 64], [0, 0, 64, 64]], [.3, .3], [5, 0])]
    check(gts, dts, 2)


def random_set(n_images, K, seed, max_gt=6, max_det=15):
    gen = torch.Generator().manual_seed(seed)
    gts, dts = [], []
    for i in range(n_images):
        ng = int(torch.randint(0, max_gt + 1, (1,), generator=gen))
        xy = torch.rand(ng, 2, generator=gen) * 600
        gb = torch.cat([xy, xy + torch.rand(ng, 2, generator=gen) * 150 + 1], 1)
        gl = torch.randint(0, K, (ng,), generator=gen)
        nd = int(torch.randint(0, max_det + 1, (1,), generator=gen))
        src = torch.randint(0, max(ng, 1), (nd,), generator=gen)
        db = (gb[src] if ng else torch.rand(nd, 4, generator=gen) * 600) + torch.randn(nd, 4, generator=gen) * 8
        dl = gl[src] if ng else torch.randint(0, K, (nd,), generator=gen)
        dl = torch.where(torch.rand(nd, generator=gen) < 0.1, torch.randint(0, K + 1, (nd,), generator=gen), dl)
        sc = torch.round(torch.rand(nd, generator=gen) * 200) / 200
        gts.append(dict(boxes=gb, labels=gl))
        dts.append(dict(boxes=db, scores=sc, labels=dl))
    return gts, dts


@pytest.mark.parametrize("K,n_images,max_det", [(2, 5000, 15), (100, 5000, 8)])
def test_seeded_random_sets(K, n_images, max_det):
    gts, dts = random_set(n_images, K, seed=K, max_det=max_det)
    check(gts, dts, K)


def test_split_updates_equal_one_update():
    gts, dts = random_set(300, 2, seed=9)
    one = evaluation.DetectionBuffer(480, 640, ["car", "pedestrian"])
    one.update(dts, gts, "dsec")
    split = evaluation.DetectionBuffer(480, 640, ["car", "pedestrian"])
    for lo in range(0, 300, 70):
        split.update(cuda(dts[lo:lo + 70]), gts[lo:lo + 70], "dsec")
    a, b = one.compute(), split.compute()
    assert a == b and a["mAP"] > 0
    ev = ref_coco.evaluate_lists(gts, dts, 2)
    assert [a["m" + k] for k in evaluation.OUT_KEYS] == ev.stats[:6].tolist()


def test_model_detections_through_detection_buffer():
    W, H, B = 240, 180, 2
    model, _ = make_model("n", H, W)
    model.cuda()
    buf = evaluation.DetectionBuffer(H, W, ["car", "pedestrian"])
    all_gt, all_dt = [], []
    gen = torch.Generator().manual_seed(3)
    for seed in (7, 8, 9):
        _, data = make_inputs(B, 5000, W, H, seed=seed, kind="clustered")
        dets = model(data.clone().cuda())[0]
        gts = []
        for x in dets:
            n = len(x["boxes"])
            keep = torch.rand(n, generator=gen) < 0.6
            bx = x["boxes"].cpu()[keep] + torch.randn(int(keep.sum()), 4, generator=gen) * 2
            extra = torch.rand(2, 2, generator=gen) * 150
            bx = torch.cat([bx, torch.cat([extra, extra + 30], 1)])
            gts.append(dict(boxes=bx, labels=torch.cat([x["labels"].cpu()[keep].long(), torch.tensor([0, 1])])))
        buf.update(dets, gts, "dsec")
        all_dt += [{k: v.cpu() for k, v in x.items()} for x in dets]
        all_gt += gts
    assert sum(len(x["boxes"]) for x in all_dt) > 0
    res = buf.compute()
    ev = ref_coco.evaluate_lists(all_gt, all_dt, 2)
    assert [res["m" + k] for k in evaluation.OUT_KEYS] == ev.stats[:6].tolist()
    check(all_gt, all_dt, 2)
