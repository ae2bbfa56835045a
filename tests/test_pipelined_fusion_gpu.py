"""PipelinedDetector with image fusion on the GPU: the image branch of step i+1 runs next to the coarse stack of step i
(per-slot branch outputs, per-slot coarse graphs), and every handle returns what model(data) returns on that batch alone,
bit for bit.

1. Consecutive hybrid batches with varying event counts and an empty sample, in TF32 and bf16, with u8 and formatted
   frames: handles resolved right away and handles resolved only after the next batch was submitted; two rounds, the
   second replaying the captured graphs.
2. The batch size and the frame shape change between batches (new geometry, new branch graphs, new coarse graphs).
3. model(data) after pipelined steps keeps its own bits: overlap is restored and the per-slot graphs stay out of the
   serial path."""
import pytest
import torch

from dagr_b200.data import EventBatch, format_data, synth_batch
from tests.helpers import make_model

pytestmark = pytest.mark.gpu

W, H = 320, 240
COUNTS = [12000, 4000, 16000, 9000, 0, 14000]          # events per sample of consecutive batches; 0: every sample empty


def _model(precision):
    model, _ = make_model("s", H, W, batch_size=2, use_image=True, img_net="resnet18")
    model.image_precision = precision
    return model.cuda()


def _batch(B, n, seed, frames, image_hw=(H, W)):
    """one formatted batch on the device; sample 1 has no events (or every sample when n == 0), frames "u8" keeps the
    loader's u8 image, "float" formats it like format_data."""
    raw = synth_batch(B, max(n, 1), W, H, seed=seed, with_image=True)
    g = torch.Generator().manual_seed(seed + 1)
    raw.image = torch.randint(0, 256, (B, 3) + tuple(image_hw), generator=g, dtype=torch.uint8)
    u8 = raw.image.clone()
    d = format_data(raw)
    keep = (d.batch != 1) & torch.full_like(d.batch, n > 0, dtype=torch.bool)
    out = EventBatch(x=d.x[keep], pos=d.pos[keep], batch=d.batch[keep], width=d.width, height=d.height,
                     time_window=d.time_window, image=u8 if frames == "u8" else d.image, num_graphs=B, dims=d.dims)
    return out.to("cuda")


def _host(dets):
    return [{k: v.cpu() for k, v in x.items()} for x in dets]


def _assert_same(want, got, what):
    assert len(want) == len(got), what
    for b, (w, r) in enumerate(zip(want, got)):
        for k in ("boxes", "scores", "labels"):
            assert w[k].dtype == r[k].dtype and torch.equal(w[k], r[k]), f"{what}: sample {b}, {k}"


def _pipelined(pd, batches, lag):
    """submit every batch; lag: handle i is resolved only after batch i+1 was submitted."""
    res, prev = [], None
    for d in batches:
        h = pd.submit(d)
        if not lag:
            res.append(h.result())
            continue
        if prev is not None:
            res.append(prev.result())
        prev = h
    if lag:
        res.append(prev.result())
    return res


def _coarse_graph_keys(eng):
    return [sw["graph"][0] for ws in eng._ws.values() for sw in ws.get("slots", {}).values() if sw.get("graph") is not None]


@pytest.mark.parametrize("frames", ["u8", "float"])
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_pipelined_hybrid_batches_equal_model_forward(precision, frames):
    from dagr_b200.pipeline import PipelinedDetector
    model = _model(precision)
    batches = [_batch(2, n, 100 + k, frames) for k, n in enumerate(COUNTS)]
    want = [_host(model(d)[0]) for d in batches]
    assert any(x["boxes"].shape[0] for w in want for x in w), "no detections at all: the comparison would be vacuous"
    pd = PipelinedDetector(model)
    for rnd in range(2):
        for lag in (False, True):
            got = _pipelined(pd, batches, lag)
            for k, (w, r) in enumerate(zip(want, got)):
                _assert_same(w, r, f"{precision} {frames} round {rnd} lag {lag} batch {k}")
    eng = model.engine
    assert eng.overlap is False
    keys = _coarse_graph_keys(eng)
    assert len(keys) == 2, "the hybrid coarse stack of each hand-off slot replays as a captured graph"
    assert {k[1] for k in keys} == {0, 1}
    br = model._image_branch
    assert {k[3] for k in br._graphs if len(k) == 4} == {0, 1}, "per-slot branch graphs"
    # 3. the serial forward after pipelined steps: own bits, its own (unslotted) branch outputs, eager coarse stack
    again = [_host(model(d)[0]) for d in batches]
    for k, (w, r) in enumerate(zip(want, again)):
        _assert_same(w, r, f"model(data) after pipelined steps, batch {k}")
    assert _coarse_graph_keys(eng) == keys, "the serial hybrid forward captures no coarse graph"
    # model(data) while pipelined handles are outstanding, then more submits (join(), the serial forward's reset of the
    # engine's output slot, fence() on the next submit)
    for rnd in range(2):                                  # at most two handles outstanding, as the contract allows
        h0, h1 = pd.submit(batches[0]), pd.submit(batches[1])
        s2 = _host(model(batches[2])[0])
        r0 = h0.result()
        h3 = pd.submit(batches[3])
        s4 = _host(model(batches[4])[0])
        r1 = h1.result()
        h5 = pd.submit(batches[5])
        got = {0: r0, 1: r1, 2: s2, 3: h3.result(), 4: s4, 5: h5.result()}
        for k, r in got.items():
            _assert_same(want[k], r, f"interleaved round {rnd} batch {k}")


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_pipelined_hybrid_batch_size_and_frame_shape_change(precision):
    from dagr_b200.pipeline import PipelinedDetector
    model = _model(precision)
    shapes = [(2, (H, W)), (2, (H, W)), (3, (H, W)), (3, (H + 32, W + 64)), (3, (H + 32, W + 64)), (2, (H, W)), (1, (H, W)),
              (2, (H, W))]
    batches = [_batch(B, COUNTS[k % len(COUNTS)] or 5000, 200 + k, "float", hw) for k, (B, hw) in enumerate(shapes)]
    want = [_host(model(d)[0]) for d in batches]
    pd = PipelinedDetector(model)
    for rnd in range(2):
        got = _pipelined(pd, batches, lag=True)
        for k, (w, r) in enumerate(zip(want, got)):
            _assert_same(w, r, f"{precision} round {rnd} batch {k} (B = {shapes[k][0]}, frame {shapes[k][1]})")
    again = [_host(model(d)[0]) for d in batches]
    for k, (w, r) in enumerate(zip(want, again)):
        _assert_same(w, r, f"model(data) after pipelined steps, batch {k}")


def test_pipelined_hybrid_precision_switch_between_batches():
    """image_precision read per submit, as model(data) reads it per call: the taps' format is part of the graph key."""
    from dagr_b200.pipeline import PipelinedDetector
    model = _model("tf32")
    batches = [_batch(2, n, 300 + k, "u8") for k, n in enumerate(COUNTS[:4])]
    plan = ["tf32", "tf32", "bf16", "bf16", "tf32", "bf16", "bf16", "tf32"]
    want = []
    for k, p in enumerate(plan):
        model.image_precision = p
        want.append(_host(model(batches[k % len(batches)])[0]))
    pd = PipelinedDetector(model)
    for rnd in range(2):
        res, prev = [], None
        for k, p in enumerate(plan):
            model.image_precision = p
            h = pd.submit(batches[k % len(batches)])
            if prev is not None:
                res.append(prev.result())
            prev = h
        res.append(prev.result())
        for k, (w, r) in enumerate(zip(want, res)):
            _assert_same(w, r, f"round {rnd} step {k} ({plan[k]})")
