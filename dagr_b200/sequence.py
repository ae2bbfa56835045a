"""Detection over a recorded sequence: many time windows of one recording as the samples of batched forwards.

    det = SequenceDetector(model, window_us=50_000, max_windows=64)
    dets = det.detect(events, t_end)                 # one dict(boxes, scores, labels) per query time, in the caller's order

Window q holds the events with t_begin[q] <= t < t_end[q], where t_begin defaults to t_end - window_us: the live window of
the streaming rings after a chunk that ends at t_end (dagr_b200.streaming), so each window's detections are the bits a
StreamingDetector would have produced at that instant.  An explicit t_begin gives anchored windows, such as the ones of
the reference's interframe evaluation (interframe_windows).

How a call runs: the recording is uploaded once (with sensor=: down-sampled, cropped and rebased once); dagr_window_bounds
finds every window's [begin, end) in the time-sorted recording; one read-back of those bounds lets the host plan blocks of
consecutive windows (plan_blocks); each block is gathered by dagr_window_gather straight into the inputs of the graph sort,
with window g of the block as sample g, and runs through Engine.forward_events + Engine.postprocess at one batch size G
(a short last block is padded with empty samples, so one geometry and one captured coarse stack serve the whole call).
The block loop has no host synchronisation; the call has two: the bounds read-back and the final result.

Image fusion: every frame a call uses runs through the model's own ImageBranch at B = 1 once, into plane arrays, and each
block passes a per-sample plane table (image_planes), so every window is sampled with its own frame as a batch of one --
the bits of the fusion streaming detectors and of model(data) at B = 1.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, ingest
from .streaming import _CameraFrames, _check_raw_frames

MAX_WINDOWS = 255                     # dagr_window_gather: G in [1, 255]
MAX_BLOCK = 1 << 24                   # dagr_window_gather / dagr_graph_sort: rows of one block < 2^24
_I32_MIN, _I32_MAX = -(1 << 31), (1 << 31) - 1


def plan_blocks(sizes, max_windows: int, max_events: int):
    """-> [(q0, q1)]: the windows of a call cut into blocks of consecutive windows, in order, each with at most max_windows
    windows and max_events events in all.  A window over max_events runs alone; one of 2^24 events or more raises
    ValueError (a block's rows are packed in 24 bits)."""
    sizes = np.asarray(sizes, dtype=np.int64).reshape(-1)
    big = np.flatnonzero(sizes >= MAX_BLOCK)
    if len(big):
        raise ValueError(f"window {int(big[0])} holds {int(sizes[big[0]])} events: a window must hold fewer than 2^24")
    blocks, q0, tot = [], 0, 0
    for q, n in enumerate(sizes.tolist()):
        if q > q0 and (q - q0 == max_windows or tot + n > max_events):
            blocks.append((q0, q))
            q0, tot = q, 0
        tot += n
    if len(sizes):
        blocks.append((q0, len(sizes)))
    return blocks


def interframe_windows(frame_t, steps: int = 10, span_us: int = 50_000):
    """the windows of the reference's interframe evaluation (scripts/run_test_interframe.py): for each n_us in
    np.linspace(0, span_us, steps) and each frame i, the window [frame_t[i], frame_t[i] + int(n_us)) read with frame i.
    Returns (t_begin, t_end, frame_idx) int64 arrays in that order (offset-major); the first window of each frame is
    empty."""
    ft = np.asarray(frame_t, dtype=np.int64).reshape(-1)
    offs = [int(n_us) for n_us in np.linspace(0, span_us, steps)]
    t_begin = np.tile(ft, len(offs))
    t_end = (ft[None, :] + np.asarray(offs, dtype=np.int64)[:, None]).reshape(-1)
    return t_begin, t_end, np.tile(np.arange(len(ft), dtype=np.int64), len(offs))


def _tensor(a, name):
    if not isinstance(a, torch.Tensor):
        a = np.ascontiguousarray(a).reshape(-1)
        if a.dtype.kind not in "iub":
            raise ValueError(f"events[{name!r}] of dtype {a.dtype}: expected integers")
        a = torch.from_numpy(a.astype(np.int64) if a.dtype.kind == "u" else a)
    a = a.reshape(-1)
    return a.to(torch.int64) if a.dtype in (torch.uint16, torch.uint32, torch.uint64) else a


def _host_i64(a, name):
    v = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    if v.dtype.kind not in "iu":
        raise ValueError(f"{name} of dtype {v.dtype}: expected integer microseconds")
    return v.astype(np.int64).reshape(-1)


class SequenceDetector:
    """Detections at many instants of one recording, computed as batched forwards.

    events: dict of x, y, t, p for one recording, host arrays or tensors (uploaded once); t non-decreasing (else
    ValueError).  Without `sensor` the events are what StreamingDetector.submit takes: x, y at the model's resolution, t in
    us within the int32 range, p the polarity -1/+1; the time base is 0.  With sensor=(width, height) they are the camera's
    raw events (t int64 us, p in {0, 1}, or +-1 with p_is_01=False): the recording is down-sampled once by
    ingest.downsample_events, in slices of at most max_events with the change map carried from slice to slice, cropped to
    y < H, and rebased to its first raw timestamp, which is what StreamingDetector(sensor=...) does to the same events fed
    from the start of the recording.  Query times are then raw times too.

    Blocks: at most max_windows windows (<= 255) and max_events gathered events each; a window over max_events runs
    alone.  Image fusion (use_image models): `frames` u8 [F, 3, H, W], or with raw_frames=True (which needs sensor=) the
    camera's u8 [F, sensor_h, sensor_w, 3], converted as the fusion streaming detectors convert them.  Window q reads the
    newest frame with frame_t <= t_end[q], or frame_idx[q] when it is given.  model.image_precision is read here, once."""

    def __init__(self, model, window_us: int = 50_000, max_windows: int = 64, max_events: int = 1 << 23, sensor=None,
                 p_is_01: bool = True, raw_frames: bool = False, device=None):
        if model.head.no_events:
            raise NotImplementedError("--no_events: the model has no event path to run over a recording")
        _check_raw_frames(raw_frames, sensor)
        self.use_image = bool(model.backbone.use_image)
        if raw_frames and not self.use_image:
            raise ValueError("raw_frames takes camera frames: it needs an image-fusion model (backbone.use_image)")
        if not 1 <= int(max_windows) <= MAX_WINDOWS:
            raise ValueError(f"max_windows={max_windows}: 1 <= max_windows <= {MAX_WINDOWS}")
        if not 1 <= int(max_events) < MAX_BLOCK:
            raise ValueError(f"max_events={max_events}: 1 <= max_events < 2^24")
        if int(window_us) < 0:
            raise ValueError(f"window_us={window_us} must be >= 0")
        self.model = model
        self.W, self.H = int(model.width), int(model.height)
        self.window_us, self.max_windows, self.max_events = int(window_us), int(max_windows), int(max_events)
        self.raw_frames = bool(raw_frames)
        self.image_precision = model.image_precision if self.use_image else None
        self.dev = torch.device(device) if device is not None else next(model.parameters()).device
        self._check_sensor(sensor, p_is_01)
        self._frame_lut = None
        self._cam = _CameraFrames(self, 0)             # frame checks and the u8 -> f32 conversion of the fusion detectors
        self.last = None

    def _check_sensor(self, sensor, p_is_01):
        self.sensor, self.p_is_01 = None, bool(p_is_01)
        if sensor is None:
            if not p_is_01:
                raise ValueError("p_is_01 describes raw sensor events: it needs sensor=(width, height)")
            return
        sw, sh = (int(v) for v in sensor)
        scale = sw // self.W
        if scale < 1 or sw != scale * self.W or sh < scale * self.H:
            raise ValueError(f"sensor {sw}x{sh} for a {self.W}x{self.H} model: the sensor width must be an integer multiple "
                             f"scale * {self.W} and the height at least scale * {self.H}")
        if sw > 1 << 16 or sh > 1 << 15:
            raise ValueError(f"sensor {sw}x{sh}: x must fit 16 bits and y 15 bits")
        self.sensor, self.scale, self.grid = (sw, sh), scale, (sw // scale, sh // scale)

    # ---- input checks (host side, before any device work) --------------------------------------------------------------
    def _check_events(self, events):
        try:
            x, y, t, p = (_tensor(events[k], k) for k in "xytp")
        except KeyError as e:
            raise ValueError(f"events needs x, y, t and p (missing {e})") from None
        n = len(t)
        if not len(x) == len(y) == len(p) == n:
            raise ValueError(f"events x, y, t, p of different lengths {len(x)}, {len(y)}, {n}, {len(p)}")
        if n >= 1 << 31:
            raise ValueError(f"{n} events: a recording holds fewer than 2^31")
        if n > 1 and bool((t[1:] < t[:-1]).any()):
            raise ValueError("events are not sorted by time (t must be non-decreasing)")
        if n and self.sensor is None and (int(t[0]) < _I32_MIN or int(t[-1]) > _I32_MAX):
            raise ValueError(f"timestamps {int(t[0])}..{int(t[-1])} us leave the int32 range (raw times need sensor=)")
        if n and self.sensor is not None:
            sw, sh = self.sensor
            if int(x.min()) < 0 or int(x.max()) >= sw or int(y.min()) < 0 or int(y.max()) >= sh:
                raise ValueError(f"event coordinates outside the {sw}x{sh} sensor")
            lo, hi = int(p.min()), int(p.max())
            if (lo < 0 or hi > 1) if self.p_is_01 else (lo < -1 or hi > 1 or int((p == 0).sum()) > 0):
                raise ValueError("polarities must be in " + ("{0, 1} (p_is_01=True)" if self.p_is_01 else "{-1, +1} (p_is_01=False)"))
            if int(t[-1]) - int(t[0]) > _I32_MAX:
                raise ValueError(f"timestamps {int(t[0])}..{int(t[-1])} us span more than the int32 range of the time base")
        return x, y, t, p

    def _check_frames(self, frames, frame_t, frame_idx, t_end):
        """-> (frame index per window, {frame index: checked frame [1, ...]}) of an image-fusion model."""
        if frames is None:
            raise ValueError("an image-fusion model needs frames")
        F = len(frames)
        if frame_idx is not None:
            fi = _host_i64(frame_idx, "frame_idx")
            if len(fi) != len(t_end):
                raise ValueError(f"{len(fi)} frame indices for {len(t_end)} windows")
            if len(fi) and (fi.min() < 0 or fi.max() >= F):
                raise ValueError(f"frame indices outside [0, {F})")
        else:
            if frame_t is None:
                raise ValueError("frames need frame_t (or a frame index per window)")
            ft = _host_i64(frame_t, "frame_t")
            if len(ft) != F:
                raise ValueError(f"{len(ft)} frame times for {F} frames")
            if len(ft) > 1 and (np.diff(ft) < 0).any():
                raise ValueError("frame_t must be sorted")
            fi = np.searchsorted(ft, t_end, side="right") - 1
            early = np.flatnonzero(fi < 0)
            if len(early):
                q = int(early[0])
                raise ValueError(f"window {q} ends at {int(t_end[q])} us, before the first frame ({int(ft[0]) if F else None})")
        return fi, {int(f): self._cam.check(frames[int(f)]) for f in np.unique(fi)}

    # ---- device work ----------------------------------------------------------------------------------------------------
    def _upload(self, x, y, t, p):
        """the recording on the device as the gather reads it (x, y int16, t int64, p int8 +-1) and its time base."""
        dev = self.dev
        x, y = x.to(dev).to(torch.int16), y.to(dev).to(torch.int16)      # uint16 and int16 share the bits below 2^15
        t, p = t.to(dev).to(torch.int64), p.to(dev).to(torch.int8)
        if self.sensor is None:
            return x.contiguous(), y.contiguous(), t.contiguous(), p.contiguous(), 0
        if self.p_is_01:
            p = (2 * p - 1).to(torch.int8)
        t_base = int(t[0]) if len(t) else 0
        (sw, sh), (ow, oh) = self.sensor, self.grid
        parts, cmap = [], None
        for a in range(0, len(t), self.max_events):
            b = a + self.max_events
            ev, cmap = ingest.downsample_events(dict(x=x[a:b], y=y[a:b], t=t[a:b], p=p[a:b]), sh, sw, oh, ow, cmap)
            parts.append(ev)
        if not parts:
            return x, y, t, p, t_base
        ev = {k: torch.cat([e[k] for e in parts]) for k in "xytp"}
        keep = ev["y"] < self.H                                           # crop, dsec_data.py:142-143
        return tuple(ev[k][keep].contiguous() for k in "xytp") + (t_base,)

    def _planes(self, fi, checked, blocks, G):
        """every frame the call uses through the model's ImageBranch at B = 1, once, into plane arrays; -> (image_feats,
        image_outs, plane table i32[blocks, G] on the device)."""
        from .model.image_branch import FrameStore, branch_of, run_frame
        m, dev = self.model, self.dev
        used = np.array(sorted(checked), dtype=np.int64)
        tab = np.zeros((len(blocks), G), dtype=np.int32)
        for i, (q0, q1) in enumerate(blocks):
            tab[i, :q1 - q0] = np.searchsorted(used, fi[q0:q1])
        if self.raw_frames and self._frame_lut is None:
            self._frame_lut = ingest.frame_lut(dev)
        store = FrameStore(len(used))
        for k, f in enumerate(used.tolist()):
            img = self._cam.to_float(checked[f].to(dev))
            run_frame(m, store, k, img, self.image_precision)
            img.record_stream(branch_of(m).stream)
        return store.feats, store.outs, torch.from_numpy(tab).to(dev)

    def _run_blocks(self, ev, begin, end, blocks, totals, G, planes):
        """the block loop: gather, forward, NMS and the copy of each block's detections, all enqueued without a host sync.
        Returns (det [Q, A, 6], ndet [Q]) on the device."""
        eng, m, lib = self.model.engine, self.model, self.model.engine.lib
        x, y, t, p, t_base = ev
        N, Q, cap = len(t), len(begin), max(max(totals), 1)
        dev = self.dev
        batch = torch.empty(cap, dtype=torch.int32, device=dev)
        pos = torch.empty((cap, 3), dtype=torch.int32, device=dev)
        feat = torch.empty(cap, dtype=torch.float32, device=dev)
        offs = torch.empty(G + 1, dtype=torch.int64, device=dev)
        feats, outs, tab = planes if planes is not None else (None, None, None)
        det_all = ndet_all = None
        for i, ((q0, q1), n) in enumerate(zip(blocks, totals)):
            eng._run("window_gather", lib.dagr_window_gather, x, y, t, p, N, begin[q0:], end[q0:], q1 - q0, int(t_base), 0, n,
                     batch, pos, feat, offs, _lib.stream_ptr())
            dec = eng.forward_events(batch[:n], pos[:n], feat[:n], G, self.W, self.H, image_feats=feats, image_outs=outs,
                                     image_planes=None if tab is None else (tab[i], 1))
            det, ndet = eng.postprocess(dec, m.conf_threshold, m.nms_threshold, self.W, self.H)
            if det_all is None:
                det_all = torch.empty((Q,) + tuple(det.shape[1:]), dtype=det.dtype, device=dev)
                ndet_all = torch.empty(Q, dtype=ndet.dtype, device=dev)
            # overlap mode: det / ndet sit in the engine's double-buffered result slots; copy them on the result stream and
            # make the copy part of the block (fence), so the slot is reused only after it
            with eng.result_stream():
                det_all[q0:q1].copy_(det[:q1 - q0])
                ndet_all[q0:q1].copy_(ndet[:q1 - q0])
            eng.fence()
        eng.join()
        return det_all, ndet_all

    @torch.no_grad()
    def detect(self, events, t_end, t_begin=None, frames=None, frame_t=None, frame_idx=None):
        """-> one dict(boxes f32[n, 4] xyxy px, scores f32[n], labels i64[n]) of CUDA tensors per window, in the caller's
        order, as model(data) returns them; `self.last` = (det f32[Q, A, 6], ndet i32[Q]) on the device, which
        utils.buffers.records_from_device turns into records.  t_end (and t_begin) int us, any order, duplicates allowed;
        t_begin defaults to t_end - window_us.  Bad input raises ValueError before any device work."""
        x, y, t, p = self._check_events(events)
        te = _host_i64(t_end, "t_end")
        tb = te - self.window_us if t_begin is None else _host_i64(t_begin, "t_begin")
        if len(tb) != len(te):
            raise ValueError(f"{len(tb)} t_begin values for {len(te)} t_end values")
        if (tb > te).any():
            raise ValueError("a window has t_begin > t_end")
        fi = checked = None
        if self.use_image:
            fi, checked = self._check_frames(frames, frame_t, frame_idx, te)
        elif frames is not None:
            raise ValueError("frames are for image-fusion models; this model is events-only")
        if self.dev.type != "cuda":
            raise RuntimeError("dagr_b200: SequenceDetector needs a CUDA device (no CPU fallback)")
        lib, dev, Q = self.model.engine.lib, self.dev, len(te)
        ev = self._upload(x, y, t, p)
        N = len(ev[2])
        begin = torch.zeros(max(Q, 1), dtype=torch.int32, device=dev)
        end = torch.zeros(max(Q, 1), dtype=torch.int32, device=dev)
        d_tb, d_te = torch.from_numpy(tb).to(dev), torch.from_numpy(te).to(dev)
        _lib.check(lib.dagr_window_bounds(ev[2], N, d_tb, d_te, Q, begin, end, _lib.stream_ptr()), "window_bounds")
        be = torch.stack([begin[:Q], end[:Q]]).cpu().numpy()                  # host sync 1: the bounds
        sizes = np.maximum(be[1].astype(np.int64) - be[0], 0)
        blocks = plan_blocks(sizes, self.max_windows, self.max_events)
        if not blocks:
            self.last = None
            return []
        G = max(q1 - q0 for q0, q1 in blocks)
        totals = [int(sizes[q0:q1].sum()) for q0, q1 in blocks]
        planes = self._planes(fi, checked, blocks, G) if self.use_image else None
        eng = self.model.engine
        eng.workspace(eng.geometry(self.W, self.H, G, dev), max(totals), dev)   # sized once: one workspace, one captured stack
        det, ndet = self._run_blocks(ev, begin, end, blocks, totals, G, planes)
        counts = ndet.cpu().tolist()                                          # host sync 2: the result
        self.last = (det, ndet)
        return [dict(boxes=det[q, :n, :4], scores=det[q, :n, 4], labels=det[q, :n, 5].long()) for q, n in enumerate(counts)]
