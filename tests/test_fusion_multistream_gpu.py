"""FusionMultiStreamDetector: S hybrid (image + events) cameras as the S samples of one streaming step, each with its own
frames, one CUDA graph for every combination of frame slots.  Every camera's image is sampled as a batch of one, so camera
s's detections must equal, bit for bit, model(data) at B = 1 over its live window with the frame frame_state(s) reports, and
a FusionStreamingDetector fed the same chunks and frames -- whatever the other cameras do.  The last test checks the four
*_planes kernels on their own at S = 6, where the batched forward's depth coordinate of sample 1 is not an exact integer."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests.test_fusion_streaming_gpu import _dense, _frames, _model
from tests.test_multistream_gpu import CHUNK, H, STEPS, W, WINDOW, _chunk, _chunks, _heterogeneous, _same, _stream, _t_end

pytestmark = pytest.mark.gpu

CHECKS = (0, 1, 2, 5, 6, 11, 12, 13, 16, 17, 20, 21, 29)     # eager (0, 1) and replayed steps, before and after the windows fill
# synced frames per camera: (step, frame index) -- both slots of every camera, switched at different steps
SCHEDULE = {0: ((0, 0), (12, 1), (21, 2)), 1: ((0, 0), (5, 1), (20, 2)), 2: ((0, 0), (16, 1))}


def _check(det, model, out, frames, s):
    fs = det.frame_state(s)
    pos, feat = det.live_window(s)
    want = _dense(model, pos, feat, frames[s][fs["frame"]])
    assert _same(out[s], want), (s, fs, len(out[s]["boxes"]), len(want["boxes"]))
    return fs


def _camera_frames(S, n=3):
    return [_frames(n, seed=30 + s) for s in range(S)]


def test_fusion_multistream_equals_dense_forward_of_each_camera():
    from dagr_b200.streaming import FusionMultiStreamDetector
    model = _model()
    evs = _heterogeneous()
    S = len(evs)
    frames = _camera_frames(S)
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    fid = [None] * S
    for k in range(STEPS):
        for s in range(S):
            for step, i in SCHEDULE[s]:
                if step == k:
                    assert det.set_frame(s, frames[s][i], t_us=k * CHUNK) == i
                    det.sync_frame(s)
                    fid[s] = (i, k * CHUNK)
        out = det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
        assert len(out) == S
        if k not in CHECKS:
            continue
        for s, ev in enumerate(evs):
            t, te = ev[2], _t_end(ev, k)
            live = (t >= te - WINDOW) & (t < te)
            st = det.window_state(s)
            assert st["live"] == int(live.sum()) and not st["overflow"], (k, s, st)
            fs = _check(det, model, out, frames, s)
            assert fs == dict(frame=fid[s][0], t_us=fid[s][1], pending=None), (k, s, fs)
    assert len(det.graphs) == 1 and det.graph is not None


def test_fusion_multistream_equals_single_camera_detectors_every_step():
    from dagr_b200.streaming import FusionMultiStreamDetector, FusionStreamingDetector
    model = _model()
    evs = _heterogeneous()
    S = len(evs)
    frames = _camera_frames(S)
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    refs = [FusionStreamingDetector(model, window_us=WINDOW, max_chunk=4096, capacity=1 << 15) for _ in range(S)]
    for k in range(STEPS):
        for s in range(S):
            for step, i in SCHEDULE[s]:
                if step == k:                              # a frame change on camera s alone
                    det.set_frame(s, frames[s][i])
                    det.sync_frame(s)
                    refs[s].set_frame(frames[s][i])
                    refs[s].sync_frame()
        out = det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
        for s, ev in enumerate(evs):
            want = refs[s].push(*_chunk(ev, k), _t_end(ev, k))[0]
            assert _same(out[s], want), (k, s, len(out[s]["boxes"]), len(want["boxes"]))
            assert det.window_state(s) == refs[s].window_state, (k, s)
            assert det.frame_state(s)["frame"] == refs[s].frame_state["frame"], (k, s)
    assert len(det.graphs) == 1


def test_fusion_multistream_frames_without_sync():
    from dagr_b200.streaming import FusionMultiStreamDetector
    model = _model()
    evs = _heterogeneous()
    S = len(evs)
    frames = _camera_frames(S, n=4)
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    with pytest.raises(RuntimeError, match="every camera"):
        det.submit(_chunks(evs, 0), [_t_end(ev, 0) for ev in evs])
    for s in range(S):
        det.set_frame(s, frames[s][0])
    sets = {0: (7, 19), 1: (10,), 2: (14, 15)}                  # camera 2: a second frame while the first may be pending
    last, seen = [0] * S, [set() for _ in range(S)]
    for k in range(STEPS):
        for s in range(S):
            if k in sets[s]:
                det.set_frame(s, frames[s][1 + sets[s].index(k)])
        if k == 22:
            det.submit(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
            assert det.set_frame(1, frames[1][2]) == 2            # two frames of camera 1 while a step is in flight
            assert det.set_frame(1, frames[1][3]) == 3
            out = det.result()
        else:
            out = det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
        for s in range(S):
            fs = _check(det, model, out, frames, s)
            assert fs["frame"] >= last[s], (k, s, fs)
            last[s] = fs["frame"]
            seen[s].add(fs["frame"])
    det.sync_frame()
    out = det.push(_chunks(evs, STEPS), [_t_end(ev, STEPS) for ev in evs])
    assert [_check(det, model, out, frames, s)["frame"] for s in range(S)] == [2, 3, 2]
    assert all(0 in x for x in seen) and len(det.graphs) == 1


def test_fusion_multistream_reset_of_one_camera_keeps_its_frame():
    from dagr_b200.streaming import FusionMultiStreamDetector
    model = _model()
    evs = _heterogeneous()
    S, R = len(evs), 12
    frames = _camera_frames(S, n=2)
    det = FusionMultiStreamDetector(model, streams=S, window_us=WINDOW, max_chunk=4096, capacity=1 << 15)
    for s in range(S):
        det.set_frame(s, frames[s][0])
    det.set_frame(1, frames[1][1])                            # camera 1 is on its second frame (slot 1) when it is reset
    det.sync_frame()
    for k in range(R):
        det.push(_chunks(evs, k), [_t_end(ev, k) for ev in evs])
    det.reset(1)
    fresh = _stream(200_000, 11, "uniform", t0=9_000_000)
    evs[1] = fresh
    out = det.push(_chunks(evs, R), [_t_end(ev, R) for ev in evs])
    assert det.window_state(1)["live"] == len(_chunk(fresh, R)[2])
    assert [det.frame_state(s)["frame"] for s in range(S)] == [0, 1, 0]
    for s in (0, 2):                                          # the other cameras keep their whole live window
        t, te = evs[s][2], _t_end(evs[s], R)
        pos, _ = det.live_window(s)
        assert np.array_equal(pos[:, 2].cpu().numpy(), t[(t >= te - WINDOW) & (t < te)]), s
    for s in range(S):
        _check(det, model, out, frames, s)


# ---- kernel level ------------------------------------------------------------------------------------------------------
def _sorted_events(eng, S, dev):
    """dagr_graph_sort of S synthetic samples: (geometry, N, start, xyb) of the B = S sort."""
    from dagr_b200 import _lib
    from dagr_b200.streaming import synth_stream
    rows = []
    for b in range(S):
        x, y, t, p = synth_stream(150_000 + 30_000 * b, 0.02, W, H, seed=40 + b, kind="clustered" if b % 2 else "uniform")
        rows.append((np.full(len(t), b), x, y, t, p))
    bt, x, y, t, p = (np.concatenate(c) for c in zip(*rows))
    N = len(t)
    batch = torch.from_numpy(bt.astype(np.int32)).to(dev)
    pos = torch.from_numpy(np.stack([x, y, t], 1).astype(np.int32)).to(dev).contiguous()
    feat = torch.from_numpy(p.astype(np.float32)).to(dev)
    geom = eng.geometry(W, H, S, dev)
    ws = eng.workspace(geom, N, dev)
    flags = torch.zeros(4, dtype=torch.int32, device=dev)
    _lib.check(eng.lib.dagr_graph_sort(C.byref(geom.c_geom), _lib.ptr(batch), _lib.ptr(pos), _lib.ptr(feat), N, _lib.ptr(ws["key"]),
                                       _lib.ptr(ws["tmp"]), _lib.ptr(ws["count"]), _lib.ptr(ws["blocksums"]), _lib.ptr(ws["start"]),
                                       _lib.ptr(ws["perm"]), _lib.ptr(ws["ti"]), _lib.ptr(ws["xyb"]), _lib.ptr(ws["feat_s"]),
                                       _lib.ptr(flags), _lib.stream_ptr()), "graph_sort")
    torch.cuda.synchronize()
    return geom, N, ws["start"], ws["xyb"]


def test_planes_kernels_equal_batch_of_one_on_each_plane():
    from dagr_b200 import _lib
    model = _model()
    eng, lib, dev = model.engine, model.engine.lib, torch.device("cuda")
    S, P = 6, 12
    table = torch.zeros((S, 4), dtype=torch.int32)
    table[:, 3] = torch.tensor([11, 0, 7, 7, 2, 5])            # a permutation with a repeated plane, in a stage-like header
    table = table.to(dev)
    pl, stride = table.view(-1)[3:], 4
    planes = table[:, 3].tolist()
    gen = torch.Generator(device=dev).manual_seed(0)
    rand = lambda *shape: torch.rand(shape, generator=gen, device=dev) * 2 - 1
    g6, N, start, xyb = _sorted_events(eng, S, dev)
    g1 = eng.geometry(W, H, 1, dev)
    st = _lib.stream_ptr()
    total = int(start[g6.NK].item())
    assert total == N
    sample = (xyb[:total].long() >> 24) & 0xff

    # dagr_l1_x0_image_planes vs dagr_l1_x0_image at B = 1 on the plane (the batch bits of xyb cleared)
    h0, w0 = 54, 80
    f0 = rand(P, 16, h0, w0)
    x0p = torch.full((2 * N * 8,), float("nan"), device=dev)
    _lib.check(lib.dagr_l1_x0_image_planes(C.byref(g6.c_geom), N, _lib.ptr(start), _lib.ptr(xyb), None, _lib.ptr(f0), h0, w0, P,
                                           _lib.ptr(pl), stride, _lib.ptr(x0p), st), "x0_image_planes")
    xyb1 = (xyb & 0xffffff).contiguous()
    for b in range(S):
        x01 = torch.full_like(x0p, float("nan"))
        f = f0[planes[b]:planes[b] + 1].contiguous()
        _lib.check(lib.dagr_l1_x0_image(C.byref(g1.c_geom), N, _lib.ptr(xyb1), None, _lib.ptr(f), h0, w0, _lib.ptr(x01), st), "x0")
        m = sample == b
        assert m.any() and torch.equal(x0p.view(2, N, 8)[:, m], x01.view(2, N, 8)[:, m]), b

    # dagr_voxel_sample_max_planes (max and mean) vs dagr_voxel_sample_max at B = 1 on the sample's voxels and plane
    h1, w1, C1, ldx, c0 = 27, 40, 64, 80, 16
    f1 = rand(P, C1, h1, w1)
    per, CP = g6.c_geom.ny1 * g6.c_geom.nx1, g6.c_geom.CP
    for mean in (0, 1):
        xg = torch.full((S * per, ldx), float("nan"), device=dev)
        _lib.check(lib.dagr_voxel_sample_max_planes(C.byref(g6.c_geom), N, _lib.ptr(start), _lib.ptr(xyb), _lib.ptr(f1), C1, h1, w1, P,
                                                    _lib.ptr(pl), stride, _lib.ptr(xg), ldx, c0, mean, st), "voxel_sample_max_planes")
        for b in range(S):
            x1 = torch.full((per, ldx), float("nan"), device=dev)
            f = f1[planes[b]:planes[b] + 1].contiguous()
            _lib.check(lib.dagr_voxel_sample_max(C.byref(g1.c_geom), N, C.c_void_p(start.data_ptr() + 4 * b * per * CP), _lib.ptr(xyb),
                                                 _lib.ptr(f), C1, h1, w1, _lib.ptr(x1), ldx, c0, mean, st), "voxel_sample_max")
            assert torch.equal(xg[b * per:(b + 1) * per, c0:], x1[:, c0:]), (mean, b)

    # dagr_sample_features_planes vs dagr_sample_features with Bi = 1 on the plane
    n, C2, h2, w2, ldo, c2 = 700, 48, 14, 20, 56, 8
    f2 = rand(P, C2, h2, w2)
    posx, posy = (rand(n) + 1) / 2, (rand(n) + 1) / 2
    bidx = torch.randint(0, S, (n,), generator=gen, device=dev, dtype=torch.int32)
    zero = torch.zeros_like(bidx)
    out = torch.full((n, ldo), float("nan"), device=dev)
    _lib.check(lib.dagr_sample_features_planes(_lib.ptr(f2), P, _lib.ptr(pl), stride, C2, h2, w2, _lib.ptr(posx), _lib.ptr(posy),
                                               _lib.ptr(bidx), n, W, H, _lib.ptr(out), ldo, c2, st), "sample_features_planes")
    for b in range(S):
        o1 = torch.full_like(out, float("nan"))
        f = f2[planes[b]:planes[b] + 1].contiguous()
        _lib.check(lib.dagr_sample_features(_lib.ptr(f), 1, C2, h2, w2, _lib.ptr(posx), _lib.ptr(posy), _lib.ptr(zero), n, W, H,
                                            _lib.ptr(o1), ldo, c2, st), "sample_features")
        m = bidx == b
        assert m.any() and torch.equal(out[m, c2:c2 + C2], o1[m, c2:c2 + C2]), b

    # dagr_head_finish_planes vs dagr_head_finish at B = 1 on the sample's cells and plane
    lv, nc = 3, 2
    L6, L1 = g6.levels[lv], g1.levels[lv]
    per = L6.nx * L6.ny
    cnt = torch.randint(0, 3, (S * per,), generator=gen, device=dev, dtype=torch.int32)
    cls, regobj = rand(S * per, nc), rand(S * per, 5)
    add_cls, add_reg, add_obj = rand(P, nc, L6.ny, L6.nx), rand(P, 4, L6.ny, L6.nx), rand(P, 1, L6.ny, L6.nx)
    dec = torch.full((S, per, 5 + nc), float("nan"), device=dev)
    _lib.check(lib.dagr_head_finish_planes(C.byref(L6.grid), _lib.ptr(cnt), _lib.ptr(cls), nc, _lib.ptr(regobj), 5, _lib.ptr(add_cls),
                                           _lib.ptr(add_reg), _lib.ptr(add_obj), nc, 32, 0, per, P, _lib.ptr(pl), stride, _lib.ptr(dec), st),
               "head_finish_planes")
    for b in range(S):
        d1 = torch.full((1, per, 5 + nc), float("nan"), device=dev)
        k, sl = planes[b], slice(b * per, (b + 1) * per)
        _lib.check(lib.dagr_head_finish(C.byref(L1.grid), _lib.ptr(cnt[sl]), _lib.ptr(cls[sl]), nc, _lib.ptr(regobj[sl]), 5,
                                        _lib.ptr(add_cls[k:k + 1]), _lib.ptr(add_reg[k:k + 1]), _lib.ptr(add_obj[k:k + 1]), nc, 32, 0, per,
                                        _lib.ptr(d1), st), "head_finish")
        assert torch.equal(dec[b], d1[0]), b
