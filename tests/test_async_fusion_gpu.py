"""Incremental updates of the image-fusion model (AsyncDAGR / forward(reset=False) with --use_image).  The reference's own
criterion (evaluate_flops.py:13-14,90,139-147, the same image for the init and the update half): after every step the
outputs equal the synchronous model(data) over all events seen so far with the stream's frame -- pooled-grid cells and
positions and the coarse edges bit-exact, grid features and decoded outputs within 1e-5, the same detections.  Also: the
xa rows of older nodes are not touched by an update, frame changes re-seed the state, a model(data) between two steps does
not disturb the stream, and with min_idx = 0 both incremental entry points give the bits of their synchronous forms."""
import ctypes as C

import pytest
import torch

from tests.helpers import assert_close, make_model

pytestmark = pytest.mark.gpu


def _data(B, n, W, H, seed=5, kind="clustered"):
    from dagr_b200.data import format_data, synth_batch
    return format_data(synth_batch(B, n, W, H, seed=seed, kind=kind, with_image=True))


def _other_image(data, seed=9):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, tuple(data.image.shape), generator=g, dtype=torch.uint8).float() / 255.0


def _with(data, sel=None, image="same"):
    from dagr_b200.data import EventBatch
    if sel is None:
        sel = torch.arange(len(data.batch))
    img = data.image if isinstance(image, str) else image
    return EventBatch(x=data.x[sel], pos=data.pos[sel], batch=data.batch[sel], width=data.width, height=data.height,
                      time_window=data.time_window, num_graphs=int(data.num_graphs), image=None if img is None else img.clone())


def _snapshot(model, dec, B):
    """what the criterion compares, taken from the last forward: decoded outputs, level-1/2 grid nodes, level-1 edges,
    detection sets."""
    from dagr_b200 import export
    L = model.engine.last
    nodes = [export.grid_nodes(L["grids"][lv], L["geom"].levels[lv], L["geom"]) for lv in range(2)]
    det, ndet = model.engine.postprocess(dec, model.conf_threshold, model.nms_threshold, model.width, model.height)
    n = ndet.tolist()
    return dict(dec=dec.clone(), nodes=[{k: nodes[lv][k].clone() for k in ("x", "pos", "cell")} for lv in range(2)],
                edges=export.grid_edges(L["grids"][0], L["geom"].levels[0]).clone(), det=[det[b, :n[b]].clone() for b in range(B)])


def _dense(model, data, B):
    """the synchronous forward (its image branch replays the same captured graphs as the stream's)."""
    dec = model.forward_decoded(data.clone().cuda())
    torch.cuda.synchronize()
    return _snapshot(model, dec, B)


def _warm(model, data):
    for _ in range(2):                                           # eager, then capture: later calls replay the branch graphs
        model.forward_decoded(data.clone().cuda())
    torch.cuda.synchronize()


def _assert_same(got, want, what):
    for lv in range(2):
        assert torch.equal(got["nodes"][lv]["cell"], want["nodes"][lv]["cell"]), f"{what}: level {lv} cells"
        assert torch.equal(got["nodes"][lv]["pos"], want["nodes"][lv]["pos"]), f"{what}: level {lv} positions"
        assert_close(got["nodes"][lv]["x"], want["nodes"][lv]["x"], tol=1e-5, what=f"async fusion level {lv} features")
    assert torch.equal(got["edges"], want["edges"]), f"{what}: level-1 edges"
    assert_close(got["dec"], want["dec"], tol=1e-5, what="async fusion decoded vs dense")
    assert [len(d) for d in got["det"]] == [len(d) for d in want["det"]], f"{what}: detection counts"
    for a, b in zip(got["det"], want["det"]):
        assert torch.equal(a[:, 5], b[:, 5]), f"{what}: labels"
        assert_close(a[:, :5], b[:, :5], tol=1e-5, what="async fusion detections")


def _split(data, B, chunks):
    """per-step index sets: every sample's (time-sorted) events cut into the same fractions / counts."""
    per_sample = [torch.nonzero(data.batch == b).flatten() for b in range(B)]
    bounds = []
    for idx in per_sample:
        if isinstance(chunks[0], float):
            cuts = (torch.tensor([0.0] + list(chunks)).cumsum(0) * len(idx)).long()
        else:
            cuts = torch.tensor([0] + list(chunks)).cumsum(0).clamp(max=len(idx))
        cuts[-1] = len(idx)
        bounds.append(cuts)
    return [torch.cat([per_sample[b][bounds[b][c]:bounds[b][c + 1]] for b in range(B)]) for c in range(len(chunks))]


CASES = [(240, 180, 1, 8000, [7999, 1], False, "n", "resnet18"),
         (640, 480, 2, 30000, [0.5, 0.2, 0.2, 0.1], False, "n", "resnet18"),     # batch planes of the 3-D grid_sample
         (320, 215, 1, 12000, [0.4, 0.3, 0.3], True, "n", "resnet18"),
         (640, 480, 1, 30000, [0.6, 0.2, 0.2], False, "s", "resnet50")]


@pytest.mark.parametrize("W,H,B,n,chunks,kto,size,img_net", CASES)
def test_async_fusion_incremental_equals_dense(W, H, B, n, chunks, kto, size, img_net):
    from dagr_b200 import export
    from dagr_b200.asynchronous import AsyncDAGR
    model, _ = make_model(size, H, W, keep_temporal_ordering=kto, use_image=True, img_net=img_net, batch_size=B)
    model.cuda()
    data = _data(B, n, W, H)
    _warm(model, data)
    steps = _split(data, B, chunks)
    a = AsyncDAGR(model)
    for c, sel in enumerate(steps):
        seen = sel if c == 0 else torch.cat([seen, sel])
        n_old = a.num_events
        old_arr = a.state.xa_arr[:n_old].clone() if c else None
        dec = a.step_decoded(_with(data, sel, image="same" if c == 0 else None).cuda(), batch_size=B)
        torch.cuda.synchronize()
        got = _snapshot(model, dec, B)
        if c:
            # older nodes: their sorted xa rows after the update are the rows they had before it, bit for bit
            L = model.engine.last
            rows = export.unsort_rows(model.engine.xa_rows(), L["ws"]["perm"], L["N"])
            assert torch.equal(rows[:n_old], old_arr), "xa rows of older nodes changed"
        want = _dense(model, _with(data, torch.sort(seen).values), B)
        _assert_same(got, want, f"step {c}")
    assert a.frames == 1
    # sliding window with the frame: evict the oldest 20 ms
    t_cut = 970000
    dec_live = a.evict_older_than(t_cut)
    torch.cuda.synchronize()
    got = _snapshot(model, dec_live, B)
    keep = torch.nonzero((model._prepare_events(data.clone().cuda())[1][:, 2] >= t_cut).cpu()).flatten()
    assert a.num_events == len(keep)
    _assert_same(got, _dense(model, _with(data, keep), B), "live window after eviction")


def _small():
    W, H, B = 320, 215, 1
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18", batch_size=B)
    model.cuda()
    data = _data(B, 12000, W, H, seed=21)
    _warm(model, data)
    return model, data, B


def test_keep_stream_drop_in_sequence_equals_forward():
    """model.keep_stream = True; model(x0, reset=True); model(x1, reset=False): the halves carry separate but equal images
    (Batch.from_data_list gives each its own copy)."""
    model, data, B = _small()
    steps = _split(data, B, [len(data.batch) - 1, 1])
    want = model(data.clone().cuda())[0]
    model.keep_stream = True
    model(_with(data, steps[0]).cuda(), reset=True)
    got = model(_with(data, steps[1]).cuda(), reset=False)[0]
    model.keep_stream = False
    assert model._async.frames == 1
    for g, w in zip(got, want):
        assert torch.equal(g["labels"], w["labels"])
        assert_close(g["boxes"], w["boxes"], tol=1e-5, what="keep_stream fusion boxes")
        assert_close(g["scores"], w["scores"], tol=1e-5, what="keep_stream fusion scores")


def test_frame_change_reseeds_and_later_steps_stay_incremental():
    from dagr_b200.asynchronous import AsyncDAGR
    model, data, B = _small()
    img2 = _other_image(data)
    steps = _split(data, B, [0.4, 0.2, 0.2, 0.2])
    a = AsyncDAGR(model)
    seen = None
    for c, sel in enumerate(steps):
        seen = sel if seen is None else torch.cat([seen, sel])
        image = {0: data.image, 1: None, 2: img2, 3: None}[c]
        dec = a.step_decoded(_with(data, sel, image=image).cuda(), batch_size=B)
        torch.cuda.synchronize()
        got = _snapshot(model, dec, B)
        frame = data.image if c < 2 else img2
        want = _dense(model, _with(data, torch.sort(seen).values, image=frame), B)
        _assert_same(got, want, f"step {c}")
    assert a.frames == 2


def test_forward_with_another_image_between_steps_does_not_disturb_the_stream():
    from dagr_b200.asynchronous import AsyncDAGR
    model, data, B = _small()
    steps = _split(data, B, [0.6, 0.4])
    want = _dense(model, data, B)
    a = AsyncDAGR(model)
    a.step_decoded(_with(data, steps[0]).cuda(), batch_size=B)
    model.forward_decoded(_with(data, image=_other_image(data, seed=13)).cuda())     # overwrites the branch's graph buffers
    dec = a.step_decoded(_with(data, steps[1], image=data.image).cuda(), batch_size=B)
    torch.cuda.synchronize()
    _assert_same(_snapshot(model, dec, B), want, "after an unrelated forward")
    assert a.frames == 1


def test_incremental_entry_points_at_min_idx_zero_equal_the_synchronous_kernels():
    """both C entry points on the inputs of a synchronous forward: conv_a_image_inc(min_idx=0) == conv_a_image_tc and
    voxel_sample_max_inc(min_idx=0) == voxel_sample_max, bit for bit; persist is seeded with the result (-inf when empty)."""
    from dagr_b200 import _lib
    W, H, B = 640, 480, 2
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18", batch_size=B)
    model.cuda()
    data = _data(B, 30000, W, H, seed=8)
    _warm(model, data)
    model.forward_decoded(data.clone().cuda())
    torch.cuda.synchronize()
    eng, L = model.engine, model.engine.last
    geom, ws, N = L["geom"], L["ws"], L["N"]
    lib, pk, g = eng.lib, eng._pack, C.byref(geom.c_geom)
    st = _lib.stream_ptr()
    P = lambda t: _lib.ptr(t)
    feats = model.last_image_feats
    x0 = ws["pool"]["x0img"]
    flags = eng._zs(ws, "flags", torch.int32)
    outs = []
    for inc in (False, True):
        xa = torch.zeros_like(ws["xa"])
        cellmask = torch.zeros(geom.cells1, dtype=torch.int32, device="cuda")
        _lib.check(lib.dagr_l1_build(g, N, P(ws["start"]), P(ws["ti"]), P(ws["xyb"]), P(ws["feat_s"]), P(geom.d_tab1), C.byref(pk["l1a_img"]),
                                     P(flags), 0, P(ws["nbr"]), P(ws["off"]), P(cellmask), P(xa), None, None, 0, st), "l1_build")
        skipv = torch.full((N, 16), float("nan"), device="cuda")
        if inc:
            _lib.check(lib.dagr_l1_conv_a_image_inc(g, N, P(ws["start"]), P(ws["xyb"]), P(ws["ti"]), P(ws["feat_s"]), P(x0), P(ws["nbr"]),
                                                    P(ws["off"]), C.byref(pk["l1img"]), P(pk["l1img_wfrag"]), 0, P(xa), P(skipv), None, None,
                                                    0, st), "conv_a_image_inc")
        else:
            _lib.check(lib.dagr_l1_conv_a_image_tc(g, N, P(ws["start"]), P(ws["xyb"]), P(ws["feat_s"]), P(x0), P(ws["nbr"]), P(ws["off"]),
                                                   C.byref(pk["l1img"]), P(pk["l1img_wfrag"]), P(xa), P(skipv), None, None, 0, st),
                       "conv_a_image_tc")
        f1 = feats[1]
        Cf = int(f1.shape[1])
        xg = torch.full((geom.cells1, 16 + Cf), float("nan"), device="cuda")
        persist = torch.full((geom.cells1, Cf), 7.0, device="cuda")
        if inc:
            _lib.check(lib.dagr_voxel_sample_max_inc(g, N, P(ws["start"]), P(ws["xyb"]), P(ws["ti"]), P(f1), Cf, int(f1.shape[2]),
                                                     int(f1.shape[3]), 0, P(persist), P(xg), 16 + Cf, 16, 0, st), "voxel_sample_max_inc")
        else:
            _lib.check(lib.dagr_voxel_sample_max(g, N, P(ws["start"]), P(ws["xyb"]), P(f1), Cf, int(f1.shape[2]), int(f1.shape[3]), P(xg),
                                                 16 + Cf, 16, 0, st), "voxel_sample_max")
        torch.cuda.synchronize()
        outs.append((xa[:2 * N * 8].clone(), skipv, xg[:, 16:].clone(), persist))
    (xa0, sk0, xg0, _), (xa1, sk1, xg1, persist) = outs
    assert torch.equal(xa1, xa0) and torch.equal(sk1, sk0)
    assert torch.equal(xg1, xg0)
    cnt = ws["grids"][0].cnt[:geom.cells1]
    occupied = cnt > 0
    assert bool(occupied.any()) and bool((~occupied).any())
    assert torch.equal(persist[occupied], xg1[occupied])
    assert bool(torch.isneginf(persist[~occupied]).all())
