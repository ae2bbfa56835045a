"""The frames the hybrid detectors keep of the image branch's outputs.

Launch lists: the C-ABI calls (Engine._run) that each consumer of frames enqueues -- FusionStreamingDetector over both frame
slots, FusionMultiStreamDetector at S = 2, AsyncDAGR (one init and one update) and SequenceDetector (one block) -- eager
steps and capture steps, in TF32 and in bf16, with the launch count of every step and the number of captured step graphs.

Frame store: frame k of a FrameStore holds, bit for bit, what the branch returned for that frame, in the taps' format
(bf16 channels_last or fp32 contiguous), for one frame of batch 2 (AsyncDAGR), two frames (the one-camera detector) and
2S frames (the multi-camera detector at S = 2)."""
import numpy as np
import pytest
import torch

from tests.helpers import make_model

pytestmark = pytest.mark.gpu

W, H = 320, 215
WINDOW, CHUNK = 20_000, 2_000
PRECISIONS = ("tf32", "bf16")


def _model(precision, B=1):
    model, _ = make_model("n", H, W, batch_size=B, use_image=True, img_net="resnet18")
    model.cuda().image_precision = precision
    return model


def _frames(n, seed=3):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (3, H, W), generator=g, dtype=torch.uint8) for _ in range(n)]


def _stream(seed):
    from dagr_b200.streaming import synth_stream
    return synth_stream(200_000, 6 * CHUNK * 1e-6, W, H, seed=seed, kind="uniform")


def _chunk(ev, k):
    x, y, t, p = ev
    a, b = np.searchsorted(t, [k * CHUNK, (k + 1) * CHUNK])
    return x[a:b], y[a:b], t[a:b], p[a:b]


class _Calls:
    """the entry points Engine._run enqueues, per step: [(launches, [name, ...]), ...]"""

    def __init__(self, monkeypatch, eng):
        from dagr_b200.engine import Engine
        self.eng, self.steps, self.names = eng, [], []
        real = Engine._run
        monkeypatch.setattr(Engine, "_run", lambda e, label, fn, *a: (self.names.append(fn.__name__), real(e, label, fn, *a))[1])

    def step(self, fn):
        self.names = []
        l0 = self.eng.launches
        out = fn()
        self.steps.append((self.eng.launches - l0, self.names))
        return out


def fusion_stream_calls(monkeypatch, precision):
    """steps 0, 1 (eager, capture) and 2 (replay) on slot 0, then a frame into slot 1: step 3 (eager + capture), 4 (replay)."""
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model(precision)
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    calls, ev, frames = _Calls(monkeypatch, model.engine), _stream(5), _frames(2)
    for k in range(5):
        if k in (0, 3):
            det.set_frame(frames[k // 3])
            det.sync_frame()
        calls.step(lambda: det.push(*_chunk(ev, k), (k + 1) * CHUNK))
    return calls.steps, len(det.graphs)


def fusion_multistream_calls(monkeypatch, precision):
    """S = 2: steps 0, 1 (eager, capture) and 2 (replay), then a new frame of camera 1 and two more replays."""
    from dagr_b200.streaming import FusionMultiStreamDetector
    model = _model(precision)
    det = FusionMultiStreamDetector(model, streams=2, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    calls, evs, frames = _Calls(monkeypatch, model.engine), [_stream(5), _stream(6)], _frames(3)
    for k in range(5):
        if k == 0:
            for s in range(2):
                det.set_frame(s, frames[s])
                det.sync_frame(s)
        if k == 3:
            det.set_frame(1, frames[2])
            det.sync_frame(1)
        calls.step(lambda: det.push([_chunk(ev, k) for ev in evs], [(k + 1) * CHUNK] * 2))
    return calls.steps, len(det.graphs)


def async_calls(monkeypatch, precision):
    """one init step with the frame and one update step."""
    from dagr_b200.asynchronous import AsyncDAGR
    from tests.test_async_fusion_gpu import _data, _split, _with
    model = _model(precision)
    data = _data(1, 6000, W, H, seed=21)
    a = AsyncDAGR(model)
    calls = _Calls(monkeypatch, model.engine)
    for c, sel in enumerate(_split(data, 1, [0.7, 0.3])):
        chunk = _with(data, sel, image=data.image if c == 0 else None).cuda()
        calls.step(lambda: a.step_decoded(chunk, batch_size=1))
    torch.cuda.synchronize()
    return calls.steps, None


def sequence_calls(monkeypatch, precision):
    """one detect() of six windows over three frames, one block."""
    from dagr_b200.sequence import SequenceDetector
    model = _model(precision)
    x, y, t, p = _stream(7)
    det = SequenceDetector(model, window_us=WINDOW, max_windows=8)
    calls = _Calls(monkeypatch, model.engine)
    frames = torch.stack(_frames(3, seed=4))
    calls.step(lambda: det.detect(dict(x=x, y=y, t=t, p=p), np.arange(1, 7) * CHUNK, frames=frames,
                                  frame_t=np.array([0, 4_000, 8_000])))
    torch.cuda.synchronize()
    return calls.steps, None


CASES = dict(fusion_stream=fusion_stream_calls, fusion_multistream=fusion_multistream_calls, async_fusion=async_calls,
             sequence=sequence_calls)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n,b", [(1, 2), (2, 1), (4, 1)])
def test_frame_store_holds_the_branch_outputs_in_their_format(monkeypatch, precision, n, b):
    from dagr_b200.model.image_branch import FrameStore, ImageBranch, run_frame
    model = _model(precision, B=b)
    returned = []
    real = ImageBranch.run

    def run(self, *a, **k):
        feats, outs, evs = real(self, *a, **k)
        torch.cuda.current_stream().wait_event(evs[1])
        returned.append(([f.clone() for f in feats], {key: [t.clone() for t in v] for key, v in outs.items()}))
        return feats, outs, evs

    monkeypatch.setattr(ImageBranch, "run", run)
    g = torch.Generator(device="cuda").manual_seed(n * 10 + b)
    store, last = FrameStore(n), {}
    for i in range(n + 2):                          # the first two runs are eager, the later ones replay the branch graphs
        run_frame(model, store, i % n, torch.rand((b, 3, H, W), generator=g, device="cuda"), precision)
        last[i % n] = returned[i]
    torch.cuda.synchronize()
    fmt = torch.channels_last if precision == "bf16" else torch.contiguous_format
    assert all(f.shape[0] == n * b and f.is_contiguous(memory_format=fmt) for f in store.feats)
    assert all(t.shape[0] == n * b and t.dtype == torch.float32 and t.is_contiguous() for v in store.outs.values() for t in v)
    for k in range(n):
        want_f, want_o = last[k]
        feats, outs = store.frame(k)
        assert all(f.shape[0] == b and f.is_contiguous(memory_format=fmt) for f in feats)
        assert all(f.dtype == a.dtype and torch.equal(f, a) for f, a in zip(feats, want_f)), k
        assert outs.keys() == want_o.keys()
        assert all(torch.equal(t, a) for key in outs for t, a in zip(outs[key], want_o[key])), k


def _coarse(sample, head):
    """the coarse stack's calls: four pooled-grid levels, image samples appended to three of them, a head on the last two"""
    level = ["grid_cat_pos", "grid_conv", "grid_linear_bn", "grid_conv"]
    pool = [sample, "grid_pool", "grid_pool_finalize"]
    return level + pool + level + pool + level + ["grid_conv"] * 4 + [head] + pool + level + ["grid_conv"] * 4 + [head]


def expected(case, precision):
    """-> ([(launches, C-ABI calls)] per step, captured step graphs) that `case` enqueues."""
    sfx = "_bf16" if precision == "bf16" else ""
    if case == "async_fusion":
        front = ["l1_build_tc", "l1_x0_image" + sfx, "l1_conv_a_image_inc", "xa_permute", "l1_conv_b_pool_voxel_tc",
                 "voxel_sample_max_inc" + sfx]
        tail = _coarse("sample_features" + sfx, "head_finish")
        steps = [(51, ["graph_sort"] + front + tail), (52, ["graph_sort", "xa_permute"] + front + tail)]
        graphs = None
    else:
        planes = "_planes" if case != "fusion_stream" else ""
        x0 = "l1_x0_image" + (planes or "_live") + sfx
        event_level = ["l1_build_tc", x0, "l1_conv_a_image_tc", "l1_conv_b_pool_voxel_tc", "voxel_sample_max" + planes + sfx]
        tail = _coarse("sample_features" + planes + sfx, "head_finish" + planes) + ["postprocess_nms"]
        sort = dict(fusion_stream=["graph_sort_ring"], fusion_multistream=["graph_sort_rings"],
                    sequence=["window_gather", "graph_sort"])[case]
        step = sort + event_level + tail
        steps = dict(fusion_stream=[step, step * 2, [], step * 2, []],           # eager, capture, replay; slot 1: capture, replay
                     fusion_multistream=[step, step * 2, [], [], []],            # one graph for every slot combination
                     sequence=[step])[case]
        steps = [(51 if case == "sequence" else 52, s) for s in steps]
        graphs = dict(fusion_stream=2, fusion_multistream=1, sequence=None)[case]
    return [(n, ["dagr_" + c for c in s]) for n, s in steps], graphs


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", list(CASES))
def test_launch_list_of_each_frame_consumer(monkeypatch, case, precision):
    steps, graphs = CASES[case](monkeypatch, precision)
    want_steps, want_graphs = expected(case, precision)
    assert graphs == want_graphs
    assert len(steps) == len(want_steps)
    for i, (got, want) in enumerate(zip(steps, want_steps)):
        assert got == want, (i, got)
