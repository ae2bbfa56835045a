"""The COCO evaluation kernels (csrc/evaluate.cu) at their internal switches, each set built by tests/eval_cases.py:
precision and recall of dagr_evaluate_bbox equal the restated COCOeval (oracle/ref_coco.py) bit for bit.

  radix sort     K = 255, 256, 257, 300 (a sixth 8-bit pass past K = 256; classes c and c + 256 differ only in the ninth
                 class bit), kept totals 2047 / 2048 / 2049 / 4097 around the 2048-item tile, equal scores over many tiles
  count scan     n_images * K past 256 * 2048, where the block-sum scan carries from one chunk to the next
  score keys     -0.0 / +0.0 in one class, +-inf, NaN (last), denormals, negative scores
  matcher        ng = 32 / 33 and kept * ng = 800 / 801 (staged fast path or recomputed slow path), a class with exactly 100
                 detections and ties across rank 100, GTs interleaved with other classes and area-ignored GTs, and GTs
                 matched at some IoU thresholds only on the slow path
  accumulation   classes with 2047 / 2048 / 2049 kept detections, a tile of only true positives and one of only false
                 positives, classes with GT only, detections only, and an empty last class
Every call gets a workspace filled with 0xFF, and two different sets run back to back in one workspace."""
import numpy as np
import pytest
import torch

from dagr_b200 import evaluation
from oracle import ref_coco
from tests import eval_cases as E
from tests.test_eval_gpu import check

pytestmark = pytest.mark.gpu


def device_eval(gts, dts, K, ws):
    """evaluation.accumulate in the caller's workspace (not cleared here)"""
    return tuple(t.cpu().numpy() for t in evaluation.accumulate(gts, dts, K, workspace=ws))


def same_bits(got, ev):
    prec, rec = got
    for name, g, w in (("precision", prec, ev.eval["precision"][..., 2]), ("recall", rec, ev.eval["recall"][..., 2])):
        bad = np.argwhere(g.view(np.int64) != w.view(np.int64))
        assert len(bad) == 0, f"{name}: {len(bad)} entries differ, first {bad[:3].tolist()}: {[(g[tuple(b)], w[tuple(b)]) for b in bad[:3]]}"


def workspace(*sets):
    need = max(evaluation.workspace_bytes(sum(len(g["boxes"]) > 0 for g in gts), K, sum(len(g["boxes"]) for g in gts),
                                          sum(len(d["boxes"]) for g, d in zip(gts, dts) if len(g["boxes"])))
               for gts, dts, K in sets)
    return torch.full((need,), 0xFF, dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("name", list(E.CASES))
def test_evaluate_bbox_at_kernel_switches(name):
    gts, dts, K = E.CASES[name]()
    ev = check(gts, dts, K)                                               # through evaluation.accumulate
    assert ev is not None
    same_bits(device_eval(gts, dts, K, workspace((gts, dts, K))), ev)    # 0xFF workspace


def test_count_scan_past_one_chunk_of_block_sums():
    gts, dts, K = E.wide_scan()
    assert sum(len(g["boxes"]) > 0 for g in gts) * K > E.SCAN_CHUNK
    ev = check(gts, dts, K)
    same_bits(device_eval(gts, dts, K, workspace((gts, dts, K))), ev)


def test_two_sets_back_to_back_in_one_workspace():
    a, b = E.CASES["acc_tiles"](), E.CASES["score_keys"]()
    ws = workspace(a, b)
    got_a = device_eval(*a, ws)
    got_b = device_eval(*b, ws)
    got_a2 = device_eval(*a, ws)
    ev_a, ev_b = ref_coco.evaluate_lists(*a), ref_coco.evaluate_lists(*b)
    same_bits(got_a, ev_a)
    same_bits(got_b, ev_b)
    same_bits(got_a2, ev_a)


def test_workspace_argument_is_checked():
    gts, dts, K = E.CASES["score_keys"]()
    ws = workspace((gts, dts, K))
    for bad in (ws[:-1], ws.view(torch.int8), ws.cpu()):
        with pytest.raises(ValueError):
            evaluation.accumulate(gts, dts, K, workspace=bad)
