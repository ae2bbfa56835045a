"""Cross-stream ordering of the overlapped paths, under forced device delays.

Under natural timing the producer of a hand-off nearly always finishes before its consumer starts, so a missing or
misplaced wait between two streams goes unnoticed.  Here one side of each hand-off is held back on the device by a spin
kernel (torch.cuda._sleep) on the stream that side runs on, and the results must still be the bits of the serial,
undelayed computation with the same weights:

1. Engine overlap, events only: PipelinedDetector steps (B = 2, with and without keep_temporal_ordering) under delays of
   the event level, the coarse stack, the forked first head scale and NMS; SequenceDetector blocks with overlap on.
2. Hybrid model(data), TF32 and bf16, eager and replayed trunk: trunk stages and coarse stack delayed, calls back to back
   with different images.
3. PipelinedDetector, hybrid: trunk stages, coarse stack and NMS delayed; the caller writes the batch in place right
   before submit (after a sleep on its own stream) and right after it; overlapped model.forward_decoded calls.
4. FusionStreamingDetector: steps while a delayed frame is pending, two set_frame calls while a delayed step reads the
   slot, two raw host frames back to back.
5. FusionMultiStreamDetector, S = 2: the same, one camera's frames changing while a delayed step reads both.
6. AsyncDAGR with frames: a model(data) on another image between two incremental steps.
7. SequenceDetector with frames.

The delays are installed with monkeypatch before a test builds its model or detector (a captured graph keeps the sleeps it
was captured with).  Each delay increments a device counter next to its sleep, so a sleep replayed inside a CUDA graph is
counted too; every test asserts that each of its delays ran at least once per step, so a renamed method or label cannot
turn it into a no-op.  The references run on a twin model (same seed, same weights) that no delay touches."""
import numpy as np
import pytest
import torch

from tests.helpers import make_model
from tests.test_async_fusion_gpu import _data as _async_data, _other_image, _split, _warm, _with
from tests.test_fusion_streaming_gpu import CHUNK, WINDOW, _chunk, _dense, _frames, _same, _stream
from tests.test_multistream_gpu import _chunks, _heterogeneous, _t_end
from tests.test_pipelined_fusion_gpu import H as PH, _assert_same, _batch, _host

pytestmark = pytest.mark.gpu

W, H = 320, 215
DELAY_MS = 15.0
SITES = ("event_late", "coarse_late", "fork_late", "nms_late", "stage1_late", "stage2_late", "copy_late", "step_late",
         "caller_late", "caller_overwrite")
ENGINE_SITES = {"event_late": "l1_conv_b_pool_voxel", "coarse_late": "cat_pos", "fork_late": "head_finish",
                "nms_late": "postprocess_nms"}

_CYCLES = {}


def _cycles_per_ms():
    """spin-kernel cycles per millisecond, timed once per session between two CUDA events (the SM clock depends on the
    card's power limit, so nothing is asserted about it)."""
    if "v" not in _CYCLES:
        torch.cuda._sleep(1000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20_000_000
        e0.record()
        torch.cuda._sleep(n)
        e1.record()
        e1.synchronize()
        _CYCLES["v"] = n / max(e0.elapsed_time(e1), 1e-3)
    return _CYCLES["v"]


def _cur():
    return torch.cuda.current_stream().cuda_stream


class Delays:
    """the delay sites `sites`, installed with monkeypatch.  Engine, ImageBranch and streaming-step sites fire only for
    the models passed to arm(); FrameStore.put has no model and fires for every store while installed."""

    def __init__(self, monkeypatch, sites, ms=DELAY_MS):
        from dagr_b200.engine import Engine
        from dagr_b200.model.image_branch import FrameStore, ImageBranch
        from dagr_b200.streaming import _RingDetector
        unknown = set(sites) - set(SITES)
        assert not unknown, unknown
        self.sites = tuple(sites)
        self.cycles = int(ms * _cycles_per_ms())
        self.hits = torch.zeros(len(SITES), dtype=torch.int64, device="cuda")
        self.models = []
        self._fresh = set()                  # engines whose coarse stack has begun and not yet reached its first cat_pos
        d = self
        if set(sites) & set(ENGINE_SITES):
            run = Engine._run

            def _run(eng, label, fn, *args):
                site = self._engine_site(eng, label)
                if site is not None:
                    st = args[-1]                             # every wrapped launch takes its stream last
                    assert (st.value or 0) == _cur(), (site, label, "the launch's stream is not the current stream")
                    d.sleep(site)
                return run(eng, label, fn, *args)

            monkeypatch.setattr(Engine, "_run", _run)
            if "coarse_late" in sites:
                coarse = Engine._coarse

                def _coarse(eng, *a, **k):
                    if d.armed(eng.model):
                        d._fresh.add(id(eng))
                    return coarse(eng, *a, **k)

                monkeypatch.setattr(Engine, "_coarse", _coarse)
        for site, name in (("stage1_late", "_stage1"), ("stage2_late", "_stage2")):
            if site in sites:
                monkeypatch.setattr(ImageBranch, name, self._branch_stage(getattr(ImageBranch, name), site))
        if "copy_late" in sites:
            put = FrameStore.put

            def _put(store, k, feats, outs):
                d.sleep("copy_late")
                return put(store, k, feats, outs)

            monkeypatch.setattr(FrameStore, "put", _put)
        if "step_late" in sites:
            enqueue = _RingDetector._enqueue

            def _enqueue(det):
                if d.armed(det.model):
                    assert _cur() == det.stream.cuda_stream, "a streaming step runs on the detector's stream"
                    d.sleep("step_late")
                return enqueue(det)

            monkeypatch.setattr(_RingDetector, "_enqueue", _enqueue)

    def _engine_site(self, eng, label):
        if not self.armed(eng.model):
            return None
        if label == "l1_conv_b_pool_voxel" and "event_late" in self.sites:
            return "event_late"
        if label == "cat_pos" and id(eng) in self._fresh:
            self._fresh.discard(id(eng))
            return "coarse_late"
        if (label == "head_finish" and "fork_late" in self.sites and eng._fstream is not None
                and _cur() == eng._fstream.cuda_stream):
            return "fork_late"
        if label == "postprocess_nms" and "nms_late" in self.sites:
            return "nms_late"
        return None

    def _branch_stage(self, fn, site):
        d = self

        def stage(br, x, precision):
            if d.armed(br.model):
                assert _cur() == br.stream.cuda_stream, f"{site}: the trunk runs on the branch's stream"
                d.sleep(site)
            return fn(br, x, precision)

        return stage

    def arm(self, model):
        self.models.append(model)
        return model

    def armed(self, model):
        return any(m is model for m in self.models)

    def sleep(self, site):
        """a spin of the configured length on the current stream, and one more count of `site` (a captured sleep counts at
        every replay)."""
        torch.cuda._sleep(self.cycles)
        self.count(site)

    def count(self, site):
        self.hits[SITES.index(site)].add_(1)

    def counts(self):
        torch.cuda.synchronize()
        return dict(zip(SITES, self.hits.tolist()))

    def check(self, steps, **least):
        """every installed site ran at least once per step: `steps` times, or least[site] times for a site that runs once per
        something else (a trunk site once per frame)."""
        c = self.counts()
        low = {s: (c[s], least.get(s, steps)) for s in self.sites if c[s] < least.get(s, steps)}
        assert not low, f"delay sites that ran fewer times than they must (ran, must): {low}"


def _twins(height=H, precision=None, **kw):
    """(reference, model to delay): the same weights, engines and image branches of their own."""
    ref, model = (make_model("s", height, W, **kw)[0].cuda() for _ in range(2))
    if precision is not None:
        ref.image_precision = model.image_precision = precision
    return ref, model


# ---- 1. Engine overlap, events only ------------------------------------------------------------------------------------
EVENTS_SITES = ["event_late", "coarse_late", "fork_late", "nms_late"]
COUNTS = [15000, 9000, 20000, 12000, 15000, 7000]


def _events_batches():
    from tests.helpers import make_inputs
    return [make_inputs(2, n, W, H, seed=31 + k, kind="uniform")[1].cuda() for k, n in enumerate(COUNTS)]


@pytest.mark.parametrize("kto", [False, True], ids=["plain", "keep_temporal_ordering"])
@pytest.mark.parametrize("sites", [[s] for s in EVENTS_SITES] + [EVENTS_SITES], ids=lambda s: "+".join(s))
def test_pipelined_events_only_under_delays(monkeypatch, sites, kto):
    from dagr_b200.pipeline import PipelinedDetector
    ref, model = _twins(keep_temporal_ordering=kto)
    batches = _events_batches()
    want = [_host(ref(d)[0]) for d in batches]
    assert any(x["boxes"].shape[0] for w in want for x in w)
    d = Delays(monkeypatch, sites)
    d.arm(model)
    pd = PipelinedDetector(model)
    steps = 0
    for rnd in range(2):                               # eager steps, then the captured per-slot coarse stacks
        prev = None
        for k, b in enumerate(batches + [None]):
            h = pd.submit(b) if b is not None else None
            if prev is not None:
                _assert_same(want[k - 1], prev.result(), f"{sites} round {rnd} batch {k - 1}")
            prev = h
        steps += len(batches)
    assert model.engine.overlap is False
    d.check(steps)


@pytest.mark.parametrize("sites", [["coarse_late"], ["nms_late"], ["coarse_late", "nms_late"]], ids=lambda s: "+".join(s))
def test_sequence_events_only_overlapped_under_delays(monkeypatch, sites):
    from dagr_b200.sequence import SequenceDetector
    from tests.test_sequence_gpu import _recording
    ref, model = _twins(batch_size=1)
    ev = _recording(300_000, 0.12, 9, "clustered")
    t_end = np.arange(4_000, 120_001, 4_000)
    want = SequenceDetector(ref, window_us=WINDOW, max_windows=7).detect(ev, t_end)
    assert sum(len(w["boxes"]) for w in want) > 0
    d = Delays(monkeypatch, sites)
    d.arm(model)
    model.engine.overlap = True
    det = SequenceDetector(model, window_us=WINDOW, max_windows=7)
    for rnd in range(3):                               # eager, warm-up and replayed coarse stacks
        got = det.detect(ev, t_end)
        bad = [q for q in range(len(t_end)) if not _same_dev(got[q], want[q])]
        assert not bad, (rnd, bad[:5])
    d.check(3 * -(-len(t_end) // 7))


def _same_dev(a, b):
    return all(torch.equal(a[k].cpu(), b[k].cpu()) for k in ("boxes", "scores", "labels"))


# ---- 2. hybrid model(data) ---------------------------------------------------------------------------------------------
HB = 2
HYBRID_COUNTS = [12000, 4000, 16000, 9000]


def _hybrid_twins(precision):
    """twins at the frame size of the hybrid batches (_batch)"""
    return _twins(PH, precision, batch_size=HB, use_image=True, img_net="resnet18")


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "replayed"])
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("sites", [["stage1_late"], ["stage2_late"], ["coarse_late"], ["fork_late"],
                                   ["stage1_late", "stage2_late", "coarse_late", "fork_late"]], ids=lambda s: "+".join(s))
def test_hybrid_forward_under_delays(monkeypatch, sites, precision, graph):
    """consecutive model.forward_decoded calls with different images, no host sync in between: the trunk of call k+1
    overwrites the branch outputs that the (delayed) coarse stack of call k reads.  The serial hybrid coarse stack is
    eager, so a delayed first head scale is joined by the stream wait alone, not by a graph capture."""
    ref, model = _hybrid_twins(precision)
    ref.image_graph = model.image_graph = graph
    batches = [_batch(HB, n, 400 + k, "float") for k, n in enumerate(HYBRID_COUNTS)]
    want = [ref.forward_decoded(b).clone() for b in batches]
    d = Delays(monkeypatch, sites)
    d.arm(model)
    got = []
    for rnd in range(2):                               # graph: two eager warm-ups, then captured branch graphs
        for b in batches:
            got.append(model.forward_decoded(b).clone())
    torch.cuda.synchronize()
    for k, g in enumerate(got):
        assert torch.equal(g, want[k % len(batches)]), f"{sites} {precision} graph={graph}: call {k}"
    dets = _host(model(batches[0])[0])
    _assert_same(_host(ref(batches[0])[0]), dets, "model(data) after the delayed calls")
    d.check(len(got) + 1)


# ---- 3. PipelinedDetector, hybrid --------------------------------------------------------------------------------------
PIPE_SITES = ["stage1_late", "stage2_late", "coarse_late", "nms_late"]


def _overwrite(dst, src):
    """write batch `src` into the tensors of batch `dst` in place, on the current stream."""
    for k in ("pos", "x", "batch", "image"):
        getattr(dst, k).copy_(getattr(src, k))


@pytest.mark.parametrize("sites,precision", [([s], "tf32") for s in PIPE_SITES] + [(PIPE_SITES, "tf32"), (PIPE_SITES, "bf16")],
                         ids=lambda v: "+".join(v) if isinstance(v, list) else v)
def test_pipelined_hybrid_under_delays(monkeypatch, sites, precision):
    from dagr_b200.pipeline import PipelinedDetector
    ref, model = _hybrid_twins(precision)
    batches = [_batch(HB, n, 500 + k, "float") for k, n in enumerate(HYBRID_COUNTS)]
    others = [_batch(HB, n, 900 + k, "float") for k, n in enumerate(HYBRID_COUNTS)]     # same shapes, other content
    want = [_host(ref(b)[0]) for b in batches]
    assert any(x["boxes"].shape[0] for w in want for x in w)
    assert all(o.pos.shape == b.pos.shape and torch.equal(o.batch, b.batch) for o, b in zip(others, batches))
    d = Delays(monkeypatch, sites)
    d.arm(model)
    pd = PipelinedDetector(model)
    steps = 0

    def lagged(make, what):
        """submit one step per batch (make(k) -> handle), resolving handle k only after step k+1 was submitted."""
        nonlocal steps
        prev = None
        for k in range(len(batches) + 1):
            h = make(k) if k < len(batches) else None
            if prev is not None:
                _assert_same(want[k - 1], prev.result(), f"{sites} {precision} {what}: batch {k - 1}")
            prev = h
        steps += len(batches)

    for rnd in range(2):                               # eager steps, then the captured branch and coarse graphs
        lagged(lambda k: pd.submit(batches[k]), f"round {rnd}")
    # caller_late: the caller's stream writes the batch after a sleep, then submits; the step must read the new content
    held = []

    def late(k):
        x = others[k].clone()
        d.sleep("caller_late")
        _overwrite(x, batches[k])
        held.append(x)
        return pd.submit(x)

    lagged(late, "caller_late")
    # caller_overwrite: right after submit returns the caller writes another valid batch into the same tensors; the step
    # has read its batch by then (the caller's stream waits for inputs_read)
    def overwrite(k):
        x = batches[k].clone()
        h = pd.submit(x)
        _overwrite(x, others[k])
        d.count("caller_overwrite")
        held.append(x)
        return h

    lagged(overwrite, "caller_overwrite")
    # overlapped model.forward_decoded without PipelinedDetector: the branch of step k + 2 reuses step k's hand-off slot
    # and must wait for step k's coarse stack, which the host never waited for
    eng = model.engine
    eng.overlap = True
    try:
        got = []
        for b in batches + batches:
            dec = model.forward_decoded(b)
            det, ndet = eng.postprocess(dec, model.conf_threshold, model.nms_threshold, model.width, model.height)
            with eng.result_stream():
                got.append((det.clone(), ndet.clone()))
        eng.join()
        torch.cuda.synchronize()
    finally:
        eng.overlap = False
    for k, (det, ndet) in enumerate(got):
        n = ndet.tolist()
        res = [dict(boxes=det[b, :n[b], :4].cpu(), scores=det[b, :n[b], 4].cpu(), labels=det[b, :n[b], 5].long().cpu())
               for b in range(HB)]
        _assert_same(want[k % len(batches)], res, f"{sites} {precision} overlapped forward {k}")
    steps += len(got)
    d.check(steps)
    c = d.counts()
    assert c["caller_late"] == len(batches) and c["caller_overwrite"] == len(batches), c


# ---- 4. FusionStreamingDetector ----------------------------------------------------------------------------------------
def _stream_twins(precision):
    return _twins(H, precision, batch_size=1, use_image=True, img_net="resnet18")


def _check_stream(det, ref, out, frames, what):
    fs = det.frame_state
    pos, feat = det.live_window()
    want = _dense(ref, pos, feat, frames[fs["frame"]])
    assert _same(out, want), (what, fs, len(out["boxes"]), len(want["boxes"]))
    return fs


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("sites", [["stage2_late"], ["copy_late"], ["stage2_late", "copy_late"]], ids=lambda s: "+".join(s))
def test_fusion_stream_steps_while_a_delayed_frame_is_pending(monkeypatch, sites, precision):
    from dagr_b200.streaming import FusionStreamingDetector
    ref, model = _stream_twins(precision)
    ev, frames = _stream(seed=9), _frames(3, seed=7)
    d = Delays(monkeypatch, sites)
    d.arm(model)
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    sets, syncs = {0: 0, 6: 1, 14: 2}, (10, 18)       # set_frame at these steps (frame 0 is never synced: the first step
    pending, steps = 0, 22                             # waits for it on the device)
    for k in range(steps):
        if k in sets:
            assert det.set_frame(frames[sets[k]], t_us=k * CHUNK) == sets[k]
        if k in syncs:
            det.sync_frame()
        out = det.push(*_chunk(ev, k), (k + 1) * CHUNK)[0]
        fs = _check_stream(det, ref, out, frames, (sites, k))
        want_frame = max(i for s, i in sets.items() if s <= k)
        if k in syncs or k == 0:
            assert fs == dict(frame=want_frame, t_us=[s for s, i in sets.items() if i == want_frame][0] * CHUNK, pending=None), (k, fs)
        else:
            assert fs["frame"] in (want_frame - 1, want_frame), (k, fs)
        if fs["pending"] is not None:
            assert fs["pending"] == fs["frame"] + 1, (k, fs)
            pending += 1
    assert pending > 0, "no step ran while a newer frame was pending: the delay did not overlap a step"
    # a detector's first frame, set while the model is warm (branch graphs captured, engine packed): the first step is
    # enqueued right away and must wait on the device for the frame it takes without a query
    fresh = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    assert fresh.set_frame(frames[2]) == 0
    out = fresh.push(*_chunk(ev, 0), CHUNK)[0]
    fs = _check_stream(fresh, ref, out, frames[2:], "first frame of a second detector")
    assert fs == dict(frame=0, t_us=None, pending=None), fs
    d.check(len(sets) + 1)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("sites", [["step_late"], ["step_late", "stage2_late", "copy_late"]], ids=lambda s: "+".join(s))
def test_fusion_stream_set_frame_twice_while_a_delayed_step_reads_the_slot(monkeypatch, sites, precision):
    """the scenario of test_fusion_stream_reset_keeps_the_frame_and_set_frame_twice with the in-flight step held back:
    the second frame's copy goes into the slot that step reads and must wait for it."""
    from dagr_b200.streaming import FusionStreamingDetector
    ref, model = _stream_twins(precision)
    ev, frames = _stream(seed=8), _frames(4, seed=6)
    d = Delays(monkeypatch, sites)
    d.arm(model)
    by_id = frames + [frames[0]]                       # frame ids 0..4: the second round sets frames 3 and 0 again
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    det.set_frame(frames[0])
    for k in range(12):
        out = det.push(*_chunk(ev, k), (k + 1) * CHUNK)[0]
        if k in (0, 1, 5, 11):
            assert _check_stream(det, ref, out, frames, k)["frame"] == 0
    det.reset()
    out = det.push(*_chunk(ev, 12), 13 * CHUNK)[0]
    assert _check_stream(det, ref, out, frames, 12)["frame"] == 0
    for rnd, (a, b) in enumerate(((1, 2), (3, 0))):    # both slots: the step in flight reads slot 0, then slot 1
        k = 13 + 3 * rnd
        det.submit(*_chunk(ev, k), (k + 1) * CHUNK)
        assert det.set_frame(frames[a]) == 2 * rnd + 1
        assert det.set_frame(frames[b]) == 2 * rnd + 2
        out = det.result()[0]
        assert _check_stream(det, ref, out, frames, k)["frame"] == 2 * rnd, "the step in flight uses the frame it started with"
        out = det.push(*_chunk(ev, k + 1), (k + 2) * CHUNK)[0]
        assert _check_stream(det, ref, out, by_id, k + 1)["frame"] in (2 * rnd + 1, 2 * rnd + 2)
        det.sync_frame()
        out = det.push(*_chunk(ev, k + 2), (k + 3) * CHUNK)[0]
        assert _check_stream(det, ref, out, by_id, k + 2)["frame"] == 2 * rnd + 2
    d.check(19, stage2_late=5, copy_late=5)           # 19 steps, five frames


def test_fusion_stream_raw_host_frames_back_to_back(monkeypatch):
    """two host frames set back to back with a delayed trunk: the pinned upload stage of the second is written while the
    first frame may still be in flight."""
    from dagr_b200.streaming import FusionStreamingDetector
    from tests.test_raw_frames_gpu import SH, SW, _prepared, _sensor_frames
    from tests.test_raw_stream_gpu import _chunk as _raw_chunk, _raw_stream, _t_end as _raw_t_end
    ref, model = _stream_twins("tf32")
    ev, raw = _raw_stream(1_000_000, seed=23, t0=50_000), _sensor_frames(4, seed=3)
    prepared = [_prepared(f) for f in raw]
    d = Delays(monkeypatch, ["stage1_late"])
    d.arm(model)
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH), raw_frames=True)
    plan = {0: (0, 1), 8: (2, 3)}                      # two host frames in a row at these steps
    pending = 0
    for k in range(16):
        for i in plan.get(k, ()):
            assert det.set_frame(raw[i]) == i
        if k == 12:
            det.sync_frame()
        out = det.push(*_raw_chunk(ev, k), t_end=_raw_t_end(ev, k))[0]
        fs = _check_stream(det, ref, out, prepared, k)
        pending += fs["pending"] is not None
        if k == 12:
            assert fs == dict(frame=3, t_us=None, pending=None), fs
    assert pending > 0, "no step ran while a newer frame was pending"
    d.check(len(raw))


# ---- 5. FusionMultiStreamDetector, S = 2 -------------------------------------------------------------------------------
@pytest.mark.parametrize("sites", [["stage2_late"], ["copy_late"], ["step_late"], ["stage2_late", "copy_late", "step_late"]],
                         ids=lambda s: "+".join(s))
def test_fusion_multistream_under_delays(monkeypatch, sites):
    from dagr_b200.streaming import FusionMultiStreamDetector
    ref, model = _stream_twins("tf32")
    evs = _heterogeneous()[:2]
    S = len(evs)
    frames = [_frames(3, seed=40 + s) for s in range(S)]
    d = Delays(monkeypatch, sites)
    d.arm(model)
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    for s in range(S):
        det.set_frame(s, frames[s][0])                 # never synced: the first step waits for both on the device
    steps, pending = 20, 0
    for k in range(steps):
        if k == 4:
            det.set_frame(0, frames[0][1])
        if k == 9:                                     # two frames of camera 1 while a step reads both cameras' slots
            det.submit(_chunks(evs, k), [_t_end(e, k) for e in evs])
            assert det.set_frame(1, frames[1][1]) == 1
            assert det.set_frame(1, frames[1][2]) == 2
            out = det.result()
        else:
            if k == 14:
                det.sync_frame()
            out = det.push(_chunks(evs, k), [_t_end(e, k) for e in evs])
        for s in range(S):
            fs = det.frame_state(s)
            pos, feat = det.live_window(s)
            want = _dense(ref, pos, feat, frames[s][fs["frame"]])
            assert _same(out[s], want), (sites, k, s, fs, len(out[s]["boxes"]), len(want["boxes"]))
            pending += fs["pending"] is not None
        if k == 9:
            assert det.frame_state(1)["frame"] == 0, "the step in flight uses the frame it started with"
        if k >= 14:
            assert [det.frame_state(s)["frame"] for s in range(S)] == [1, 2], k
    if set(sites) & {"stage2_late", "copy_late"}:
        assert pending > 0, "no step ran while a newer frame was pending"
    d.check(steps, stage2_late=5, copy_late=5)        # five frames through the trunk and into the store


# ---- 6. AsyncDAGR with frames ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sites", [["coarse_late"], ["stage2_late"], ["coarse_late", "stage2_late"]], ids=lambda s: "+".join(s))
def test_async_fusion_under_delays(monkeypatch, sites):
    from dagr_b200.asynchronous import AsyncDAGR

    def run(model):
        data = _async_data(1, 12000, W, H, seed=21)
        _warm(model, data)
        steps = _split(data, 1, [0.5, 0.25, 0.25])
        a = AsyncDAGR(model)
        out = [a.step_decoded(_with(data, steps[0]).cuda(), batch_size=1).clone()]
        model.forward_decoded(_with(data, image=_other_image(data, seed=13)).cuda())     # overwrites the branch's outputs
        out.append(a.step_decoded(_with(data, steps[1], image=data.image).cuda(), batch_size=1).clone())
        out.append(a.step_decoded(_with(data, steps[2], image=None).cuda(), batch_size=1).clone())
        torch.cuda.synchronize()
        assert a.frames == 1
        return out

    ref, model = _stream_twins("tf32")
    want = run(ref)
    d = Delays(monkeypatch, sites)
    d.arm(model)
    got = run(model)
    for k, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"{sites}: step {k}"
    d.check(len(got))


# ---- 7. SequenceDetector with frames -----------------------------------------------------------------------------------
@pytest.mark.parametrize("sites", [["stage2_late"], ["copy_late"], ["stage2_late", "copy_late"]], ids=lambda s: "+".join(s))
def test_sequence_with_frames_under_delays(monkeypatch, sites):
    from dagr_b200.sequence import SequenceDetector
    from tests.test_sequence_gpu import _dense as _window_dense, _frames as _seq_frames, _recording
    ref, model = _stream_twins("tf32")
    ev = _recording(300_000, 0.12, 10, "uniform")
    frame_t = np.array([0, 40_000, 80_000])
    frames = _seq_frames(len(frame_t), (3, H, W), seed=5)
    t_end = np.arange(4_000, 120_001, 8_000)
    d = Delays(monkeypatch, sites)
    d.arm(model)
    model.engine.overlap = True
    det = SequenceDetector(model, window_us=WINDOW, max_windows=4)
    for rnd in range(2):
        got = det.detect(ev, t_end, frames=frames, frame_t=frame_t)
        for q, te in enumerate(t_end):
            a, b = np.searchsorted(ev["t"], [te - WINDOW, te])
            f = frames[np.searchsorted(frame_t, te, side="right") - 1]
            want = _window_dense(ref, ev["x"][a:b], ev["y"][a:b], ev["t"][a:b], ev["p"][a:b], f)
            assert _same_dev(got[q], want), (sites, rnd, q)
    d.check(2 * len(frame_t))
