"""End to end, the shipped configurations no other test runs: image fusion at dagr-m and dagr-l (the layer inputs
(162, 96), (194, 96), (194, 128) and (258, 128)), the resnet34 image trunk, and the stream bench.py measures -- dagr-l at
640 x 480 through StreamingDetector.  The forwards are checked against the oracle as in tests/test_gpu_parity.py; the
stream's detections against the synchronous forward over its live window, bit for bit."""
import numpy as np
import pytest
import torch

from tests.helpers import make_model
from tests.test_gpu_parity import _check_forward

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("size,img_net", [("m", "resnet18"), ("l", "resnet18"), ("s", "resnet34")])
def test_image_fusion_parity_vs_oracle_at_shipped_sizes(size, img_net):
    from dagr_b200.data import format_data, synth_batch
    W, H, B = 240, 180, 2
    model, args = make_model(size, H, W, use_image=True, img_net=img_net, batch_size=B)
    model.cuda()
    raw = synth_batch(B, 5000, W, H, seed=79, kind="clustered", with_image=True, ragged=True)
    _check_forward(model, args, format_data(raw.clone()), B, H, W, image=True, check_public=False)


def test_benchmarked_stream_equals_dense_forward_on_live_window():
    """bench.py's streaming configuration (the model of stream_benchmark: dagr-l, randomised BN, 640 x 480, a uniform
    1 Mevents/s stream of seed 99, 50 ms live window, max_chunk 4096) in 2.5 ms chunks.  The detections of the eager
    steps, of the replayed steps and of the steps after evictions equal model(live window) exactly."""
    from dagr_b200.data import EventBatch
    from dagr_b200.streaming import StreamingDetector, synth_stream
    W, H = 640, 480
    model, args = make_model("l", H, W, batch_size=1)
    model.cuda()
    window_us, chunk_us, total_us = 50_000, 2_500, 80_000
    x, y, t, p = synth_stream(1_000_000, total_us * 1e-6, W, H, seed=99, kind="uniform")
    det = StreamingDetector(model, window_us=window_us, max_chunk=4096)
    bounds = np.searchsorted(t, np.arange(0, total_us + chunk_us, chunk_us))
    checked = 0
    for k in range(len(bounds) - 1):
        a, b = int(bounds[k]), int(bounds[k + 1])
        t_end = (k + 1) * chunk_us
        out = det.push(x[a:b], y[a:b], t[a:b], p[a:b], t_end)
        if k in (0, 1, 2, 9, 19, 20, 21, 26, 31):
            st = det.window_state
            live = (t >= t_end - window_us) & (t < t_end)
            assert st["live"] == int(live.sum()) and not st["overflow"], (k, st, int(live.sum()))
            if k >= 20:
                assert st["evicted"] > 0
            pos, feat = det.live_window()
            assert np.array_equal(pos[:, 2].cpu().numpy(), t[live])
            n = len(feat)
            d = EventBatch(x=feat.view(-1, 1).clone(), pos=torch.zeros(n, 3, device="cuda"), batch=torch.zeros(n, dtype=torch.long, device="cuda"),
                           width=torch.tensor([W]), height=torch.tensor([H]), time_window=torch.tensor([1_000_000]),
                           pos_denorm=pos.clone(), num_graphs=1, dims=(W, H, 1_000_000))
            want = model(d)[0][0]
            assert len(want["boxes"]) > 0
            assert len(out[0]["boxes"]) == len(want["boxes"]), (k, len(out[0]["boxes"]), len(want["boxes"]))
            assert torch.equal(out[0]["boxes"], want["boxes"].cpu()) and torch.equal(out[0]["scores"], want["scores"].cpu())
            assert torch.equal(out[0]["labels"], want["labels"].cpu())
            checked += 1
    assert checked == 9 and det.graph is not None
