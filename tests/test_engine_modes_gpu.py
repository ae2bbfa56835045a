"""The launches of each Engine.forward_events mode that tests/test_frame_store_gpu.py does not pin.

For every step the test records the (profile label, C-ABI entry point) pairs Engine._run enqueues, in order, and the
launch count: the plain events-only forward at B = 2, serial and overlapped, each through its eager, capture and replay
steps; keep_node_features; keep_temporal_ordering, plain and incremental; StreamingDetector; MultiStreamDetector at
S = 2; events-only AsyncDAGR (one init step, one update step); and the hybrid plain forward in fp32 and bf16."""
import numpy as np
import pytest
import torch

from tests.helpers import make_inputs, make_model

pytestmark = pytest.mark.gpu

W, H = 320, 215
WINDOW, CHUNK = 20_000, 2_000


class _Calls:
    """the (label, entry point) pairs Engine._run enqueues, per step: [(launches, [(label, name), ...]), ...]"""

    def __init__(self, monkeypatch, eng):
        from dagr_b200.engine import Engine
        self.eng, self.steps, self.calls = eng, [], []
        real = Engine._run
        monkeypatch.setattr(Engine, "_run", lambda e, label, fn, *a: (self.calls.append((label, fn.__name__)),
                                                                      real(e, label, fn, *a))[1])

    def step(self, fn):
        self.calls = []
        l0 = self.eng.launches
        out = fn()
        self.steps.append((self.eng.launches - l0, self.calls))
        return out


def _batch(B=2, n=12_000, seed=31):
    return make_inputs(B, n, W, H, seed=seed, kind="uniform")[1].cuda()


def plain(monkeypatch, overlap=False, steps=3, **over):
    model, _ = make_model("n", H, W, **over)
    model.cuda()
    eng = model.engine
    eng.overlap = overlap
    calls, d = _Calls(monkeypatch, eng), _batch()
    for _ in range(steps):
        calls.step(lambda: model.forward_decoded(d))
    eng.join()
    torch.cuda.synchronize()
    return calls.steps


def node_features(monkeypatch):
    model, _ = make_model("n", H, W)
    model.cuda().engine.keep_node_features = True
    calls = _Calls(monkeypatch, model.engine)
    calls.step(lambda: model.forward_decoded(_batch()))
    return calls.steps


def asynchronous(monkeypatch, **over):
    """one init step on 70 % of every sample's events, one update step on the rest."""
    from dagr_b200.asynchronous import AsyncDAGR
    from tests.test_async_fusion_gpu import _split, _with
    model, _ = make_model("n", H, W, **over)
    model.cuda()
    data = make_inputs(2, 12_000, W, H, seed=5, kind="clustered")[1]
    a = AsyncDAGR(model)
    calls = _Calls(monkeypatch, model.engine)
    for sel in _split(data, 2, [0.7, 0.3]):
        chunk = _with(data, sel, image=None).cuda()
        calls.step(lambda: a.step_decoded(chunk, batch_size=2))
    torch.cuda.synchronize()
    return calls.steps


def _stream(seed):
    from dagr_b200.streaming import synth_stream
    return synth_stream(200_000, 4 * CHUNK * 1e-6, W, H, seed=seed, kind="uniform")


def _chunk(ev, k):
    x, y, t, p = ev
    a, b = np.searchsorted(t, [k * CHUNK, (k + 1) * CHUNK])
    return x[a:b], y[a:b], t[a:b], p[a:b]


def streaming(monkeypatch):
    from dagr_b200.streaming import StreamingDetector
    model, _ = make_model("n", H, W)
    det = StreamingDetector(model.cuda(), window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    calls, ev = _Calls(monkeypatch, model.engine), _stream(5)
    for k in range(3):
        calls.step(lambda: det.push(*_chunk(ev, k), (k + 1) * CHUNK))
    return calls.steps


def multistream(monkeypatch):
    from dagr_b200.streaming import MultiStreamDetector
    model, _ = make_model("n", H, W)
    det = MultiStreamDetector(model.cuda(), streams=2, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    calls, evs = _Calls(monkeypatch, model.engine), [_stream(5), _stream(6)]
    for k in range(3):
        calls.step(lambda: det.push([_chunk(ev, k) for ev in evs], [(k + 1) * CHUNK] * 2))
    return calls.steps


def hybrid(monkeypatch, precision):
    from tests.test_async_fusion_gpu import _data
    model, _ = make_model("n", H, W, batch_size=2, use_image=True, img_net="resnet18")
    model.cuda().image_precision = precision
    d = _data(2, 12_000, W, H, seed=21).cuda()
    calls = _Calls(monkeypatch, model.engine)
    calls.step(lambda: model.forward_decoded(d))
    torch.cuda.synchronize()
    return calls.steps


CASES = dict(serial=plain, overlapped=lambda mp: plain(mp, overlap=True, steps=6), node_features=node_features,
             temporal=lambda mp: plain(mp, steps=1, keep_temporal_ordering=True), async_events=asynchronous,
             async_temporal=lambda mp: asynchronous(mp, keep_temporal_ordering=True), streaming=streaming,
             multistream=multistream, hybrid_tf32=lambda mp: hybrid(mp, "tf32"), hybrid_bf16=lambda mp: hybrid(mp, "bf16"))


def _conv(lv, cin, cout):
    return (f"grid_conv_L{lv}_{cin}x{cout}", "dagr_grid_conv")


def _coarse(image=None, temporal=False, dense=False):
    """the coarse stack of dagr-n: layer2..5 with pool2..4, a head scale on the last two levels.  image: the entry-point
    suffix of sample_features for a hybrid model (its taps widen the layer inputs), None for events-only."""
    cin = (82, 98, 66, 66) if image is not None else (18, 66, 34, 34)
    cout = (64, 32, 32, 32)
    out = []

    def level(k):
        out.extend([("cat_pos", "dagr_grid_cat_pos"), _conv(k + 1, cin[k], cout[k]), ("linear_bn", "dagr_grid_linear_bn"),
                    _conv(k + 1, cout[k], cout[k])])

    def pool():
        out.extend(([("sample_features", "dagr_sample_features" + image)] if image is not None else [])
                   + [("grid_pool", "dagr_grid_pool"), ("grid_pool_finalize", "dagr_grid_pool_finalize")]
                   + ([("temporal_filter", "dagr_grid_temporal_filter")] if temporal else []))

    def head(lv):
        out.extend([_conv(lv, 32, 32), _conv(lv, 32, 64), _conv(lv, 32, 2), _conv(lv, 32, 5), ("head_finish", "dagr_head_finish")]
                   + ([("to_dense", "dagr_grid_to_dense")] * 3 if dense else []))

    level(0); pool(); level(1); pool(); level(2); head(3); pool(); level(3); head(4)
    return out


SORT = ("graph_sort", "dagr_graph_sort")
BUILD = ("l1_build", "dagr_l1_build_tc")
CONV_B = ("l1_conv_b_pool_voxel", "dagr_l1_conv_b_pool_voxel_tc")
GATHER, SCATTER = ("xa_gather", "dagr_xa_permute"), ("xa_scatter", "dagr_xa_permute")
FILTER = ("temporal_filter", "dagr_grid_temporal_filter")
NMS = ("postprocess_nms", "dagr_postprocess_nms")


def expected(case):
    """[(launches, [(label, entry point), ...]) per step] that `case` enqueues.  A capture step records the coarse stack
    twice (eager, then captured) and counts it once; a replay records the eager launches alone but counts the graph's."""
    events, coarse = [SORT, BUILD, CONV_B], _coarse()
    if case in ("serial", "overlapped"):
        # 1 prepare_events + 10 event-level kernels + 32 coarse kernels per step; the overlapped steps alternate two slots
        per_slot = [events + coarse, events + coarse * 2, events]
        return [(43, s) for s in (per_slot if case == "serial" else [s for s in per_slot for _ in range(2)])]
    if case == "node_features":
        return [(49, events + _coarse(dense=True))]
    if case == "temporal":
        return [(47, events + [FILTER] + _coarse(temporal=True))]
    if case in ("async_events", "async_temporal"):
        t = case == "async_temporal"
        tail = [SCATTER, CONV_B] + [FILTER] * t + _coarse(temporal=t)
        return [(44 + 4 * t, [SORT, BUILD] + tail), (45 + 4 * t, [SORT, GATHER, BUILD] + tail)]
    if case in ("streaming", "multistream"):
        # 2 stream_push[_multi] kernels (counted by the detector) + 10 + 32 + NMS; eager, capture, replay
        sort = ("graph_sort", "dagr_graph_sort_ring" + ("s" if case == "multistream" else ""))
        step = [sort, BUILD, CONV_B] + coarse + [NMS]
        return [(45, step), (45, step * 2), (45, [])]
    sfx = "_bf16" if case == "hybrid_bf16" else ""
    # 1 prepare_events + 6 + 2 + x0 1 + conv_a 2 + conv_b 2 + voxel max 1 + 35 coarse (three samples more)
    return [(50, [SORT, BUILD, ("l1_x0_image", "dagr_l1_x0_image" + sfx), ("l1_conv_a_image", "dagr_l1_conv_a_image_tc"),
                  CONV_B, ("voxel_sample_max", "dagr_voxel_sample_max" + sfx)] + _coarse(image=sfx))]


@pytest.mark.parametrize("case", list(CASES))
def test_launch_list_of_each_mode(monkeypatch, case):
    steps, want = CASES[case](monkeypatch), expected(case)
    assert len(steps) == len(want)
    for i, (got, w) in enumerate(zip(steps, want)):
        assert got == w, (i, got)
