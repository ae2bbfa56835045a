"""COCO bbox evaluation without a GPU: the restated COCOeval (oracle/ref_coco.py) against the golden fixture made with the
reference's own buffers.py / coco_eval.py, hand-computed AP values, and the C-ABI surface of dagr_evaluate_bbox."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from dagr_b200 import _lib, evaluation
from oracle import ref_coco

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = np.load(Path(__file__).parent / "golden" / "coco_eval_golden.npz")


def golden_case(name):
    n = int(GOLDEN[f"{name}_n"])
    t = lambda k: torch.from_numpy(GOLDEN[k])
    dets = [dict(boxes=t(f"{name}_det{i}_boxes"), scores=t(f"{name}_det{i}_scores"), labels=t(f"{name}_det{i}_labels")) for i in range(n)]
    gts = [dict(boxes=t(f"{name}_gt{i}_boxes"), labels=t(f"{name}_gt{i}_labels")) for i in range(n)]
    return gts, dets, int(GOLDEN[f"{name}_K"])


def oracle_stats(gts, dets, K):
    ev = ref_coco.evaluate_lists(gts, dets, K)
    return [0.0] * 6 if ev is None else [float(v) for v in ev.stats[:6]]


@pytest.mark.parametrize("name", ["k2", "k5", "nodet", "nogt"])
def test_oracle_equals_reference_plumbing(name):
    keys = [str(k) for k in GOLDEN[f"{name}_keys"]]
    assert keys == sorted("m" + k for k in evaluation.OUT_KEYS)
    want = dict(zip(keys, GOLDEN[f"{name}_stats"].tolist()))
    got = dict(zip(("m" + k for k in evaluation.OUT_KEYS), oracle_stats(*golden_case(name))))
    assert got == want


def d(boxes, scores, labels):
    return dict(boxes=torch.tensor(boxes, dtype=torch.float32).reshape(-1, 4), scores=torch.tensor(scores, dtype=torch.float32),
                labels=torch.tensor(labels, dtype=torch.int64))


def g(boxes, labels):
    return dict(boxes=torch.tensor(boxes, dtype=torch.float32).reshape(-1, 4), labels=torch.tensor(labels, dtype=torch.int64))


def test_kat_perfect_detections_give_one():
    gts = [g([[10, 10, 60, 60], [100, 100, 300, 300]], [0, 1]), g([[5, 5, 20, 20]], [0])]
    dts = [d([[10, 10, 60, 60], [100, 100, 300, 300]], [.9, .8], [0, 1]), d([[5, 5, 20, 20]], [.5], [0])]
    s = oracle_stats(gts, dts, 2)
    assert s[:3] == [1.0, 1.0, 1.0]
    # one small GT (15 x 15): its single TP has pr = 1 / (1 + eps); class 1 has no small GT -> excluded
    assert s[3] == 1 / (1 + np.spacing(1))
    assert s[4] == 1 / (1 + np.spacing(1)) and s[5] == 1 / (1 + np.spacing(1))


def test_kat_false_positive_ranked_above_true_positive():
    # one GT; FP at 0.9, TP at 0.8: pr = [0, 1/2], envelope [1/2, 1/2], rc = [0, 1] -> q = 1/2 at every recall threshold
    gts = [g([[0, 0, 100, 100]], [0])]
    dts = [d([[200, 200, 300, 300], [0, 0, 100, 100]], [.9, .8], [0, 0])]
    ev = ref_coco.evaluate_lists(gts, dts, 1)
    half = 1 / (2 + np.spacing(1))
    assert np.all(ev.eval["precision"][:, :, 0, 0, 2] == half)
    assert ev.stats[0] == half


def test_kat_gt_matched_at_exactly_one_threshold():
    # IoU = 20 * 7 / (2 * 30 * 7 - 20 * 7) = 0.5 exactly: a TP at iouThrs[0] only
    gts = [g([[0, 0, 30, 7]], [0])]
    dts = [d([[10, 0, 40, 7]], [.7], [0])]
    ev = ref_coco.evaluate_lists(gts, dts, 1)
    p = ev.eval["precision"][:, :, 0, 0, 2]
    one = 1 / (1 + np.spacing(1))                        # a single TP: pr = 1 / (1 + eps)
    assert np.all(p[0] == one) and np.all(p[1:] == 0.0)
    assert ev.stats[1] == np.mean([one] * 101) and ev.stats[2] == 0.0 and ev.stats[0] == np.mean([one] * 101 + [0.0] * 909)


def test_kat_class_without_gt_is_excluded():
    gts = [g([[0, 0, 100, 100]], [0])]
    dts = [d([[0, 0, 100, 100], [0, 0, 50, 50]], [.9, .8], [0, 1])]
    ev = ref_coco.evaluate_lists(gts, dts, 2)
    assert np.all(ev.eval["precision"][:, :, 1, :, 2] == -1)
    assert ev.stats[0] == np.mean([1 / (1 + np.spacing(1))] * 1010)   # the mean skips class 1
    assert ev.stats[3] == -1.0                           # no small GT at all


def test_kat_no_detections_gives_zeros():
    gts = [g([[0, 0, 100, 100]], [0])]
    assert oracle_stats(gts, [d([], [], [])], 2) == [0.0] * 6
    assert evaluation.evaluate_detection(gts, [d([], [], [])]) == {k: 0.0 for k in evaluation.OUT_KEYS}
    # detections only in images without GT are never counted
    assert evaluation.evaluate_detection([g([], [])], [d([[0, 0, 1, 1]], [1.], [0])]) == {k: 0.0 for k in evaluation.OUT_KEYS}


def test_summarize_matches_oracle_on_its_precision():
    gts, dets, K = golden_case("k5")
    ev = ref_coco.evaluate_lists(gts, dets, K)
    s = evaluation.summarize(ev.eval["precision"][..., 2])
    assert [s[k] for k in evaluation.OUT_KEYS] == ev.stats[:6].tolist()


def test_compute_without_gpu_raises(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    buf = evaluation.DetectionBuffer(240, 304, ["car", "pedestrian"])
    buf.update([d([[0, 0, 10, 10]], [.5], [0])], [g([[0, 0, 10, 10]], [0])], "dsec")
    with pytest.raises(RuntimeError):
        buf.compute()
    with pytest.raises(RuntimeError):
        evaluation.evaluate_detection([g([[0, 0, 10, 10]], [0])], [d([[0, 0, 10, 10]], [.5], [0])])


def test_shims_export_the_evaluation():
    from dagr.utils.buffers import DetectionBuffer
    from dagr.utils.coco_eval import evaluate_detection
    assert DetectionBuffer is evaluation.DetectionBuffer and evaluate_detection is evaluation.evaluate_detection


def test_eval_symbols_exported_declared_and_sized():
    header = (ROOT / "include" / "dagr_b200.h").read_text()
    lib = _lib.load()
    for name in ("dagr_eval_workspace_bytes", "dagr_evaluate_bbox"):
        assert name in _lib.EXPORTS and re.search(rf"\b{name}\s*\(", header) and hasattr(lib, name)
    assert lib.dagr_abi_version() == 3
    small = evaluation.workspace_bytes(10, 2, 30, 100)
    assert small % 256 == 0 and small > 0
    # 40 bytes per detection row (two key and value buffers, four flag words) dominate at scale
    big = evaluation.workspace_bytes(100_000, 2, 500_000, 17_500_000)
    assert 40 * 17_500_000 < big < 44 * 17_500_000
    assert evaluation.workspace_bytes(10, 2, 30, 200) > small
    for bad in ((0, 2, 1, 1), (10, 0, 1, 1), (10, 70000, 1, 1), (10, 2, 1, -1)):
        with pytest.raises(RuntimeError):
            evaluation.workspace_bytes(*bad)


# ---- the case builders of tests/eval_cases.py (the sets tests/test_eval_kernels_gpu.py runs) -----------------------------
def test_eval_case_builders_reach_the_kernel_switches():
    from tests import eval_cases as E
    for n in (2047, 2048, 2049, 4097):
        gts, dts, K = E.CASES[f"kept_{n}"]()
        assert E.kept_total(gts, dts, K) == n
        assert sum(len(d["boxes"]) for d in dts) > n                      # some detections are dropped
    gts, dts, K = E.CASES["equal_scores_many_tiles"]()
    assert E.kept_total(gts, dts, K) > 5 * E.RS_TILE and torch.cat([d["scores"] for d in dts]).unique().tolist() == [0.5]
    for K in (255, 256, 257, 300):
        gts, dts, k = E.CASES[f"radix_k{K}"]()
        labels = torch.cat([d["labels"] for d in dts])
        assert k == K and int(labels.max()) == K - 1 and (K <= 256 or int(labels.min()) >= 256)
    for name, pair in (("radix_k257_bit8", (0, 256)), ("radix_k300_bit8", (43, 299))):
        counts = E.class_counts(*E.CASES[name]())
        assert counts[pair[0]] > 0 and counts[pair[1]] > 0
    for ng, nk in ((32, 25), (32, 26), (33, 10), (8, 100), (9, 89)):
        gts, dts, _ = E.CASES[f"match_ng{ng}_nk{nk}"]()
        assert int((gts[0]["labels"] == 0).sum()) == ng and E.class_counts(gts, dts, 2)[0] == nk
    fast = {(ng, nk): ng <= 32 and ng * nk <= E.EV_IOU_CAP for ng, nk in ((32, 25), (32, 26), (33, 10), (8, 100), (9, 89))}
    assert fast == {(32, 25): True, (32, 26): False, (33, 10): False, (8, 100): True, (9, 89): False}
    gts, dts, K = E.CASES["rank_ties"]()
    assert sorted(len(d["boxes"]) for d in dts) == [100, 101, 102, 130, 140]
    for d in dts:
        s = np.sort(d["scores"].numpy())[::-1]
        if len(s) > 100:
            assert s[99] == s[100] or s[100] == s[101]                        # a tie straddles the cut at 100
    counts = E.class_counts(*E.CASES["acc_tiles"]())
    assert counts.tolist()[:4] == [E.AC_TILE - 1, E.AC_TILE, E.AC_TILE + 1, 2 * E.AC_TILE + 5]
    assert counts[4] == 0 and counts[5] == 30 and counts[6] == 0
    gts, _, _ = E.CASES["acc_tiles"]()
    glab = torch.cat([g["labels"] for g in gts])
    assert int((glab == 4).sum()) > 0 and int((glab == 5).sum()) == 0 and int((glab == 6).sum()) == 0
    gts, dts, _ = E.CASES["slow_path_thresholds"]()
    assert len(gts[0]["boxes"]) > 32


def test_eval_case_score_keys_and_oracle_order():
    from tests import eval_cases as E
    gts, dts, K = E.score_keys()
    s = torch.cat([d["scores"] for d in dts]).numpy()
    bits = s.view(np.uint32)
    assert np.isnan(s).any() and np.isposinf(s).any() and np.isneginf(s).any() and (s < 0).any()
    assert (bits == 0x80000000).any() and (bits == 0).any()                # -0.0 and +0.0
    assert ((bits & 0x7F800000) == 0).sum() > (bits & 0x7FFFFFFF == 0).sum()   # denormals
    # numpy's order, which the device's score key restates: -0.0 ties +0.0, NaN last
    assert list(ref_coco._order([-0.0, 0.0, np.nan, 1.0, np.inf])) == [4, 3, 0, 1, 2]
    ev = ref_coco.evaluate_lists(gts, dts, K)
    assert ev is not None and ev.stats[0] > 0


def test_eval_case_wide_scan_passes_one_chunk():
    from tests import eval_cases as E
    gts, dts, K = E.wide_scan()
    assert len(gts) * K > E.SCAN_CHUNK and all(len(g["boxes"]) == 1 for g in gts)
    assert len(set(torch.cat([d["labels"] for d in dts]).tolist())) == K
