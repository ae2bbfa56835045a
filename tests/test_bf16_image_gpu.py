"""bf16 image branch (DAGR.image_precision = "bf16") on the GPU.

1. Every bf16 NHWC sampling kernel returns, bit for bit, what its fp32 NCHW form returns on the fp32 upcast of the same map.
2. forward_events fed the bf16 taps equals forward_events fed the same taps upcast to fp32 NCHW, bit for bit.
3. In bf16 mode the entry points agree under the contracts the tf32 tests use: the streaming detectors equal model(data)
   bit for bit, AsyncDAGR within 1e-5, raw frames equal host-prepared ones, --no_events runs.
4. The default is untouched: tf32 outputs keep their bits after a bf16 run, and a load_state_dict after the bf16 capture
   reaches the bf16 copy.
5. The precision cost of bf16 against tf32 on seeded config-3 inputs, printed and bounded."""
import ctypes as C

import pytest
import torch

from tests.helpers import make_model, rel_err
from tests.test_fusion_multistream_gpu import SCHEDULE, _camera_frames, _sorted_events
from tests.test_fusion_streaming_gpu import _dense, _frames
from tests.test_multistream_gpu import CHUNK, H, STEPS, W, WINDOW, _chunk, _chunks, _heterogeneous, _same, _stream, _t_end

pytestmark = pytest.mark.gpu


def _model(precision="bf16", **over):
    model, _ = make_model("s", H, W, batch_size=1, use_image=True, img_net="resnet18", **over)
    model.image_precision = precision
    return model.cuda()


def _pair(shape, gen):
    """a bf16 map in NHWC (channels_last [n, C, h, w]) and its fp32 NCHW upcast"""
    m = (torch.rand(shape, generator=gen, device="cuda") * 4 - 2).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    return m, m.float().contiguous()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _eq(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))       # bits, NaN included


# ---- 1. kernels ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 3])
def test_bf16_kernels_equal_fp32_forms_on_the_upcast_map(B):
    from dagr_b200 import _lib
    model = _model()
    eng, lib, dev = model.engine, model.engine.lib, torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(B)
    g, N, start, xyb = _sorted_events(eng, B, dev)                      # events on the whole sensor, its border included
    gp = C.byref(g.c_geom)
    st = _lib.stream_ptr()
    ti = eng.workspace(g, N, dev)["ti"]
    P = 2 * B + 1
    table = torch.tensor([(3 * b + 1) % P for b in range(B)], dtype=torch.int32, device=dev)

    # x0: plain, live (ring capacity above the live total) and planes; odd h, w
    h0, w0 = 107, 161
    for maps, planes in ((_pair((B, 16, h0, w0), gen), False), (_pair((P, 16, h0, w0), gen), True)):
        mb, mf = maps
        if planes:
            a, b = _nan(2 * N * 8), _nan(2 * N * 8)
            _lib.check(lib.dagr_l1_x0_image_planes(gp, N, _lib.ptr(start), _lib.ptr(xyb), None, _lib.ptr(mf), h0, w0, P, _lib.ptr(table), 1,
                                                   _lib.ptr(a), st), "x0 planes")
            _lib.check(lib.dagr_l1_x0_image_planes_bf16(gp, N, _lib.ptr(start), _lib.ptr(xyb), None, _lib.ptr(mb), 16, h0, w0, P,
                                                        _lib.ptr(table), 1, _lib.ptr(b), st), "x0 planes bf16")
            assert _eq(a, b), "x0 planes"
            continue
        a, b = _nan(2 * N * 8), _nan(2 * N * 8)
        _lib.check(lib.dagr_l1_x0_image(gp, N, _lib.ptr(xyb), None, _lib.ptr(mf), h0, w0, _lib.ptr(a), st), "x0")
        _lib.check(lib.dagr_l1_x0_image_bf16(gp, N, _lib.ptr(xyb), None, _lib.ptr(mb), 16, h0, w0, _lib.ptr(b), st), "x0 bf16")
        assert _eq(a, b), "x0 plain"
        cap = N + 777
        xyb_cap = torch.zeros(cap, dtype=xyb.dtype, device=dev)
        xyb_cap[:N] = xyb[:N]
        a, b = _nan(2 * cap * 8), _nan(2 * cap * 8)
        _lib.check(lib.dagr_l1_x0_image_live(gp, cap, _lib.ptr(start), _lib.ptr(xyb_cap), None, _lib.ptr(mf), h0, w0, _lib.ptr(a), st), "x0 live")
        _lib.check(lib.dagr_l1_x0_image_live_bf16(gp, cap, _lib.ptr(start), _lib.ptr(xyb_cap), None, _lib.ptr(mb), 16, h0, w0, _lib.ptr(b), st),
                   "x0 live bf16")
        assert _eq(a, b) and not torch.isnan(a.view(2, cap, 8)[:, :N]).any(), "x0 live"

    # voxel max / mean: plain, inc (min_idx 0, then > 0) and planes; staged windows (C = 64 fast path, C = 48 general path)
    # and windows too large for shared memory (C = 128 at the sensor's resolution)
    cells = g.cells1
    ldx, c0 = 144, 16
    for C1, h1, w1 in ((64, 53, 81), (48, 27, 41), (128, H, W + 1)):
        mb, mf = _pair((B, C1, h1, w1), gen)
        pb, pf = _pair((P, C1, h1, w1), gen)
        for mean in (0, 1):
            a, b = _nan(cells, ldx), _nan(cells, ldx)
            _lib.check(lib.dagr_voxel_sample_max(gp, N, _lib.ptr(start), _lib.ptr(xyb), _lib.ptr(mf), C1, h1, w1, _lib.ptr(a), ldx, c0, mean, st),
                       "voxel")
            _lib.check(lib.dagr_voxel_sample_max_bf16(gp, N, _lib.ptr(start), _lib.ptr(xyb), _lib.ptr(mb), C1, h1, w1, _lib.ptr(b), ldx, c0,
                                                      mean, st), "voxel bf16")
            assert _eq(a, b), ("voxel", C1, mean)
            a, b = _nan(cells, ldx), _nan(cells, ldx)
            _lib.check(lib.dagr_voxel_sample_max_planes(gp, N, _lib.ptr(start), _lib.ptr(xyb), _lib.ptr(pf), C1, h1, w1, P, _lib.ptr(table), 1,
                                                        _lib.ptr(a), ldx, c0, mean, st), "voxel planes")
            _lib.check(lib.dagr_voxel_sample_max_planes_bf16(gp, N, _lib.ptr(start), _lib.ptr(xyb), _lib.ptr(pb), C1, h1, w1, P,
                                                             _lib.ptr(table), 1, _lib.ptr(b), ldx, c0, mean, st), "voxel planes bf16")
            assert _eq(a, b), ("voxel planes", C1, mean)
        pa, pbf = _nan(cells, C1), _nan(cells, C1)
        for min_idx in (0, N // 2):
            a, b = _nan(cells, ldx), _nan(cells, ldx)
            _lib.check(lib.dagr_voxel_sample_max_inc(gp, N, _lib.ptr(start), _lib.ptr(xyb), _lib.ptr(ti), _lib.ptr(mf), C1, h1, w1, min_idx,
                                                     _lib.ptr(pa), _lib.ptr(a), ldx, c0, 0, st), "voxel inc")
            _lib.check(lib.dagr_voxel_sample_max_inc_bf16(gp, N, _lib.ptr(start), _lib.ptr(xyb), _lib.ptr(ti), _lib.ptr(mb), C1, h1, w1,
                                                          min_idx, _lib.ptr(pbf), _lib.ptr(b), ldx, c0, 0, st), "voxel inc bf16")
            assert _eq(a, b) and _eq(pa, pbf), ("voxel inc", C1, min_idx)

    # sample_features: plain (Bi = B) and planes; nodes on the map border and beyond it
    n, C2, h2, w2, ldo, c2 = 900, 64, 15, 21, 80, 16
    posx, posy = torch.rand(n, generator=gen, device=dev), torch.rand(n, generator=gen, device=dev)
    posx[:8] = torch.tensor([0.0, 1.0, 0.0, 1.0, (W - 1) / W, 0.5, 1.02, -0.01], device=dev)
    posy[:8] = torch.tensor([0.0, 0.0, 1.0, 1.0, (H - 1) / H, 1.0, 0.5, 0.5], device=dev)
    bidx = torch.randint(0, B, (n,), generator=gen, device=dev, dtype=torch.int32)
    mb, mf = _pair((B, C2, h2, w2), gen)
    a, b = _nan(n, ldo), _nan(n, ldo)
    _lib.check(lib.dagr_sample_features(_lib.ptr(mf), B, C2, h2, w2, _lib.ptr(posx), _lib.ptr(posy), _lib.ptr(bidx), n, W, H, _lib.ptr(a),
                                        ldo, c2, st), "sample")
    _lib.check(lib.dagr_sample_features_bf16(_lib.ptr(mb), B, C2, h2, w2, _lib.ptr(posx), _lib.ptr(posy), _lib.ptr(bidx), n, W, H,
                                             _lib.ptr(b), ldo, c2, st), "sample bf16")
    assert _eq(a, b), "sample_features"
    pb, pf = _pair((P, C2, h2, w2), gen)
    a, b = _nan(n, ldo), _nan(n, ldo)
    _lib.check(lib.dagr_sample_features_planes(_lib.ptr(pf), P, _lib.ptr(table), 1, C2, h2, w2, _lib.ptr(posx), _lib.ptr(posy),
                                               _lib.ptr(bidx), n, W, H, _lib.ptr(a), ldo, c2, st), "sample planes")
    _lib.check(lib.dagr_sample_features_planes_bf16(_lib.ptr(pb), P, _lib.ptr(table), 1, C2, h2, w2, _lib.ptr(posx), _lib.ptr(posy),
                                                    _lib.ptr(bidx), n, W, H, _lib.ptr(b), ldo, c2, st), "sample planes bf16")
    assert _eq(a, b), "sample_features planes"
    torch.cuda.synchronize()


# ---- 2. event path isolated from the trunk --------------------------------------------------------------------------------
def _data(B, n, w=W, h=H, seed=5):
    from dagr_b200.data import format_data, synth_batch
    return format_data(synth_batch(B, n, w, h, seed=seed, kind="clustered", with_image=True))


def test_forward_events_on_bf16_taps_equals_their_fp32_upcast():
    B = 2
    model, _ = make_model("s", H, W, batch_size=B, use_image=True, img_net="resnet18")
    model.cuda().image_precision = "bf16"
    data = _data(B, 20000).cuda()
    model(data.clone())
    feats = [f.clone() for f in model.last_image_feats]
    outs = {k: [t.clone() for t in v] for k, v in model.last_image_outs.items()}
    assert all(f.dtype == torch.bfloat16 and f.is_contiguous(memory_format=torch.channels_last) for f in feats)
    assert all(t.dtype == torch.float32 and t.is_contiguous() for v in outs.values() for t in v)
    batch_i, pos_i, feat, w, h = model._prepare_events(data.clone())
    eng = model.engine
    got = eng.forward_events(batch_i, pos_i, feat, B, w, h, image_feats=feats, image_outs=outs).clone()
    want = eng.forward_events(batch_i, pos_i, feat, B, w, h, image_feats=[f.float().contiguous() for f in feats], image_outs=outs)
    assert _eq(got, want)
    with pytest.raises(ValueError, match="all float32 or all bfloat16"):
        eng.forward_events(batch_i, pos_i, feat, B, w, h, image_feats=[feats[0].float()] + feats[1:], image_outs=outs)
    with pytest.raises(ValueError, match="channels_last"):
        eng.forward_events(batch_i, pos_i, feat, B, w, h, image_feats=[f.contiguous() for f in feats], image_outs=outs)


# ---- 3. entry points in bf16 mode ----------------------------------------------------------------------------------------
def test_bf16_fusion_stream_equals_dense_forward_with_its_frame():
    from dagr_b200.streaming import FusionStreamingDetector
    model = _model()
    ev = _stream(300_000, 5, "clustered")
    frames = _frames(3)
    det = FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    model.image_precision = "tf32"                                    # read at construction: no effect on the detector
    assert det.image_precision == "bf16"
    at = {0: (0, True), 10: (1, True), 20: (2, False)}                # step: (frame, synced)
    for k in range(STEPS):
        if k in at:
            i, sync = at[k]
            assert det.set_frame(frames[i], t_us=k) == i
            if sync:
                det.sync_frame()
            else:
                torch.cuda.synchronize()                              # the step promotes it with its event query
        out = det.push(*_chunk(ev, k), _t_end(ev, k))[0]
        if k not in (0, 1, 2, 5, 10, 11, 12, 20, 21, 29):
            continue
        fs = det.frame_state
        pos, feat = det.live_window()
        model.image_precision = "bf16"
        want = _dense(model, pos, feat, frames[fs["frame"]])
        model.image_precision = "tf32"
        assert _same(out, want), (k, fs, len(out["boxes"]), len(want["boxes"]))
        slot = det._slots[det._cur][0]
        assert all(f.dtype == torch.bfloat16 and f.is_contiguous(memory_format=torch.channels_last) for f in slot)
    assert set(det.graphs) == {0, 1} and det.frame_state["frame"] == 2


def test_bf16_fusion_multistream_equals_dense_forward_of_each_camera():
    from dagr_b200.streaming import FusionMultiStreamDetector
    model = _model()
    evs = _heterogeneous()
    S = len(evs)
    frames = _camera_frames(S)
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    for k in range(STEPS):
        for s in range(S):
            for step, i in SCHEDULE[s]:
                if step == k:
                    det.set_frame(s, frames[s][i], t_us=k)
                    det.sync_frame(s)
        out = det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
        if k not in (0, 1, 2, 5, 12, 13, 16, 17, 21, 29):
            continue
        for s in range(S):
            fs = det.frame_state(s)
            pos, feat = det.live_window(s)
            want = _dense(model, pos, feat, frames[s][fs["frame"]])
            assert _same(out[s], want), (k, s, fs)
    pf = det._planes[0]
    assert all(f.dtype == torch.bfloat16 and f.shape[0] == 2 * S and f.is_contiguous(memory_format=torch.channels_last) for f in pf)
    assert len(det.graphs) == 1


def test_bf16_async_incremental_steps_and_frame_change_match_dense():
    from dagr_b200.asynchronous import AsyncDAGR
    from tests.test_async_fusion_gpu import _assert_same, _dense as _dense_snap, _other_image, _split, _warm, _with
    B = 1
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18", batch_size=B)
    model.cuda().image_precision = "bf16"
    data = _data(B, 12000, seed=21)
    _warm(model, data)
    img2 = _other_image(data)
    a = AsyncDAGR(model)
    seen = None
    for c, sel in enumerate(_split(data, B, [0.4, 0.2, 0.2, 0.2])):
        seen = sel if seen is None else torch.cat([seen, sel])
        image = {0: data.image, 1: None, 2: img2, 3: None}[c]
        dec = a.step_decoded(_with(data, sel, image=image).cuda(), batch_size=B)
        torch.cuda.synchronize()
        from tests.test_async_fusion_gpu import _snapshot
        got = _snapshot(model, dec, B)
        want = _dense_snap(model, _with(data, torch.sort(seen).values, image=data.image if c < 2 else img2), B)
        _assert_same(got, want, f"bf16 step {c}")
    assert a.frames == 2 and a._feats[0].dtype == torch.bfloat16


def test_bf16_raw_frames_equal_host_prepared_frames():
    from dagr_b200.streaming import FusionStreamingDetector
    from tests.test_raw_frames_gpu import SH, SW, _raw_stream, _sensor_frames, _set
    from tests.test_raw_frames_gpu import H as RH, W as RW, WINDOW as RWIN, _chunk as _rchunk, _t_end as _rt_end
    model, _ = make_model("s", RH, RW, batch_size=1, use_image=True, img_net="resnet18")
    model.cuda().image_precision = "bf16"
    ev, frames = _raw_stream(1_000_000, seed=21, t0=77_000), _sensor_frames(3, seed=1)
    kw = dict(window_us=RWIN, max_chunk=8192, capacity=1 << 15, sensor=(SW, SH))
    det = FusionStreamingDetector(model, raw_frames=True, **kw)
    ref = FusionStreamingDetector(model, **kw)
    for k in range(14):
        if k in (0, 5, 10):
            _set(det, ref, frames[k // 5], device=k == 5, sync=k != 10)
        c = _rchunk(ev, k)
        out = det.push(*c, t_end=_rt_end(ev, k))[0]
        want = ref.push(*c, t_end=_rt_end(ev, k))[0]
        assert _same(out, want) and det.frame_state == ref.frame_state, k
    assert det._slots[det._cur][0][0].dtype == torch.bfloat16


def test_bf16_no_events_runs():
    model, _ = make_model("n", H, W, batch_size=2, use_image=True, img_net="resnet18", no_events=True)
    model.cuda().image_precision = "bf16"
    data = _data(2, 3000).cuda()
    for _ in range(3):                                                # eager, capture, replay
        dets = model(data.clone())[0]
    assert len(dets) == 2 and all(torch.isfinite(d["boxes"]).all() for d in dets)
    assert model.last_image_feats[0].dtype == torch.bfloat16


# ---- 4. the default is untouched -----------------------------------------------------------------------------------------
def _decoded(model, data, n=3):
    for _ in range(n):                                                # eager, capture, replay
        dec = model.forward_decoded(data.clone())
    return dec.clone()


def test_tf32_bits_survive_a_bf16_run_and_reload_reaches_the_bf16_copy():
    B = 2
    data = _data(B, 15000, seed=8).cuda()
    model, _ = make_model("s", H, W, batch_size=B, use_image=True, img_net="resnet18")
    model.cuda()
    never, _ = make_model("s", H, W, batch_size=B, use_image=True, img_net="resnet18")
    never.cuda()
    tf32_before = _decoded(model, data)
    model.image_precision = "bf16"
    bf16 = _decoded(model, data)
    assert not _eq(bf16, tf32_before)
    model.image_precision = "tf32"
    assert _eq(_decoded(model, data), tf32_before)
    assert _eq(_decoded(never, data), tf32_before)
    # new weights after the bf16 capture: bf16 outputs become those of a fresh bf16 model built with them
    other, _ = make_model("s", H, W, seed=3, batch_size=B, use_image=True, img_net="resnet18")
    sd = other.state_dict()
    model.load_state_dict(sd)
    model.image_precision = "bf16"
    fresh, _ = make_model("s", H, W, batch_size=B, use_image=True, img_net="resnet18")
    fresh.load_state_dict(sd)
    fresh.cuda().image_precision = "bf16"
    reloaded = _decoded(model, data)
    assert not _eq(reloaded, bf16)
    assert _eq(reloaded, _decoded(fresh, data))
    # an in-place weight change (no load_state_dict) is caught by the engine's weight key
    with torch.no_grad():
        for p in model.backbone.net.parameters():
            p.mul_(0.5)
    assert not _eq(_decoded(model, data), reloaded)


# ---- 5. precision cost, reported -----------------------------------------------------------------------------------------
def _iou(a, b):
    lt = torch.max(a[:, None, :2], b[None, :, :2])
    rb = torch.min(a[:, None, 2:4], b[None, :, 2:4])
    inter = (rb - lt).clamp(min=0).prod(-1)
    area = lambda x: (x[:, 2] - x[:, 0]).clamp(min=0) * (x[:, 3] - x[:, 1]).clamp(min=0)
    return inter / (area(a)[:, None] + area(b)[None, :] - inter).clamp(min=1e-9)


def bf16_precision_report(B=2, seed=0):
    """bf16 against tf32 on seeded config-3 inputs (dagr-s + ResNet-50, 640x480, random weights with randomised BN)."""
    model, _ = make_model("s", 480, 640, seed=seed, batch_size=B, use_image=True, img_net="resnet50")
    model.cuda()
    data = _data(B, 60000, w=640, h=480, seed=11 + seed).cuda()
    rep = {}
    res = {}
    for prec in ("tf32", "bf16"):
        model.image_precision = prec
        dec = _decoded(model, data)
        feats = [f.float().clone() for f in model.last_image_feats]
        det, ndet = model.engine.postprocess(dec, model.conf_threshold, model.nms_threshold, model.width, model.height)
        res[prec] = (dec, feats, [det[b, :n].clone() for b, n in enumerate(ndet.tolist())])
    (d32, f32, k32), (d16, f16, k16) = res["tf32"], res["bf16"]
    rep["taps_max_rel"] = [float((a - b).abs().max() / b.abs().max()) for a, b in zip(f16, f32)]
    rep["taps_mean_rel"] = [float((a - b).abs().mean() / b.abs().mean()) for a, b in zip(f16, f32)]
    rep["decoded_max_rel"] = rel_err(d16, d32)                      # |a - b| / (|b| + mean|b|), max over elements
    rep["decoded_mean_rel"] = float(((d16 - d32).abs() / (d32.abs() + d32.abs().mean())).mean())
    matched = total = 0
    for a, b in zip(k32, k16):
        total += len(a)
        if len(a) and len(b):
            ok = (_iou(a[:, :4], b[:, :4]) >= 0.5) & (a[:, None, 5] == b[None, :, 5])
            matched += int(ok.any(1).sum())
    rep["detections_tf32"], rep["detections_bf16"] = total, sum(len(b) for b in k16)
    rep["matched_share"] = matched / total if total else 1.0
    return rep


def test_bf16_precision_against_tf32_is_bounded():
    rep = bf16_precision_report()
    print("bf16 vs tf32:", rep)
    # bounds from the H100 measurement (taps <= 2.1e-2 max / 1.2e-2 mean relative, decoded 0.40 max softened / 2.7e-3 mean,
    # 20 % of the tf32 detections matched): random weights leave the detections on near-equal scores, so the matched share
    # is fragile and says little about a trained model
    assert max(rep["taps_max_rel"]) < 0.04 and max(rep["taps_mean_rel"]) < 0.02, rep
    assert rep["decoded_max_rel"] < 0.6 and rep["decoded_mean_rel"] < 0.006, rep
    assert rep["detections_tf32"] > 0 and rep["matched_share"] >= 0.1, rep
