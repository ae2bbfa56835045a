"""Continuous streaming detection (BASELINE.json configs[4]: one ~1 Mevents/s stream per GPU, 1 ms chunks, 50 ms live window).

What the reference offers for this: `SlidingWindowGraph` with a `min_index` watermark (src/dagr/graph/ev_graph.py:121-136,
ev_graph.cu:62) that the model never uses, and an asynchronous engine that can do ONE update after its initialisation
(SURVEY section 0, fact 4).  The contract here is the one a consumer needs: after every chunk the detections equal the
synchronous forward over the live window (events with t >= t_chunk_end - window), exactly.

How a step works (everything on the device, ONE CUDA graph replay per chunk, no host synchronisation inside):

  pinned stage --H2D--> dagr_stream_push      evicts the window's prefix older than t_cut by moving the ring's head
                                              (binary search over the time-sorted ring, O(log n), no data movement) and
                                              appends the chunk behind the tail
               --> dagr_graph_sort_ring       cell-major counting sort of the live window read through the ring
               --> k_l1_build / k_l1_conv_b2  event level (launches cover the ring capacity; the live count is device data)
               --> coarse stack, head, NMS    fixed-shape launches
               --D2H--> pinned detections

MultiStreamDetector runs S such streams (S cameras) as the S samples of ONE step: S rings, a packed stage, and
dagr_stream_push_multi / dagr_graph_sort_rings in place of the single-ring calls; everything below the sort already
works on a batch.  The step is still one CUDA graph replay.

FusionStreamingDetector streams the hybrid (image + events) model: a camera frame runs through the image trunk once, into one
of two frame slots, and every chunk's step (one replay of that slot's graph) reads the newest frame whose trunk has finished.
FusionMultiStreamDetector does the same for S hybrid cameras in one step: the frame slots of all cameras are planes of one
array, and each camera's plane travels in its stage header, so one graph serves every combination of slots.

Why the event level is recomputed over the window instead of patched: evicting an event changes the neighbour lists of
every node it fed (the K cap admits the next candidate of the spiral), i.e. of the window's oldest 10 ms -- and their
activations feed the next 10 ms.  At 50 k live events the per-voxel kernels take ~0.1 ms for the WHOLE window
(they are built for 2.4 M events per launch), less than bookkeeping a change set would; the append-only incremental
path (only new events probed / convolved, `min_idx`) remains available in dagr_b200.asynchronous for the reference's
own init + update criterion.
"""
from __future__ import annotations

import time

import numpy as np
import torch

from . import _lib


RING_CTL = 8                          # ints per stream in a control block (DAGR_RING_CTL)
MAX_STREAMS = 127                     # dagr_stream_push_multi: 1 <= S <= 127
MAX_RING_SLOTS = 1 << 24              # S * capacity < 2^24: sorted positions are packed in 24 bits


def _pow2_at_least(n: int) -> int:
    cap = 1
    while cap < n:
        cap <<= 1
    return cap


class _RingDetector:
    """What StreamingDetector and MultiStreamDetector share: the device rings of `streams` x `cap` slots, a pinned stage
    and its device copy, and the step itself -- H2D of the stage, push, forward over the live windows, NMS, D2H of the
    detections and of the control block.  The first two steps run eagerly (they allocate every buffer of the step); the
    second is followed by one capture, and every later step is one replay of that CUDA graph.  A detector whose steps read
    different buffers (FusionStreamingDetector's two frame slots) keeps one graph per _graph_key(); a key first used after
    the warm-up is captured right after its first (eager) step."""

    def _setup(self, model, streams: int, window_us: int, max_chunk: int, capacity: int, device):
        self.model, self.eng = model, model.engine
        self.lib = self.eng.lib
        self.W, self.H = int(model.width), int(model.height)
        self.window_us, self.max_chunk = int(window_us), int(max_chunk)
        self.cap = _pow2_at_least(capacity)
        dev = torch.device(device) if device is not None else next(model.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("dagr_b200: streaming needs a CUDA device (no CPU fallback)")
        self.dev = dev
        n = streams * self.cap
        self.batch = torch.zeros(n, dtype=torch.int32, device=dev)
        self.pos = torch.zeros((n, 3), dtype=torch.int32, device=dev)
        self.feat = torch.zeros(n, dtype=torch.float32, device=dev)
        nstage = 4 * streams + 4 * streams * self.max_chunk
        self.stage_h = torch.zeros(nstage, dtype=torch.int32).pin_memory()
        self.stage_d = torch.zeros(nstage, dtype=torch.int32, device=dev)
        self._stage_np = self.stage_h.numpy()
        self.stream = torch.cuda.Stream(device=dev)
        self.graphs = {}                      # _graph_key() -> captured step
        self._res_h = None
        self._done = None
        self._warm = 0

    @property
    def graph(self):
        """the captured step (None until the second step has run)."""
        return self.graphs.get(0)

    def _graph_key(self):
        """which captured step the next step replays (a step graph bakes in every pointer it reads)."""
        return 0

    def _image_inputs(self):
        """(image_feats, image_outs) of the next step: None for the events-only model."""
        return None, None

    def _image_planes(self):
        """(plane table, stride) when image_feats / image_outs are per-stream plane arrays (forward_events), else None."""
        return None

    def _push(self):
        raise NotImplementedError

    def _enqueue(self):
        """one streaming step on the current stream (eager or under capture)."""
        m, eng = self.model, self.eng
        self.stage_d.copy_(self.stage_h, non_blocking=True)
        self._push()
        eng.launches += 2
        feats, outs = self._image_inputs()
        dec = eng.forward_events(self.batch, self.pos, self.feat, self._B, self.W, self.H, image_feats=feats, image_outs=outs,
                                 ring=self.ctl, ring_streams=self._ring_streams, image_planes=self._image_planes())
        det, ndet = eng.postprocess(dec, m.conf_threshold, m.nms_threshold, self.W, self.H)
        if self._res_h is None:
            self._res_h = (torch.empty(det.shape, dtype=det.dtype).pin_memory(), torch.empty(ndet.shape, dtype=ndet.dtype).pin_memory(),
                           torch.empty(self.ctl.shape, dtype=torch.int32).pin_memory())
        self._res_h[0].copy_(det, non_blocking=True)
        self._res_h[1].copy_(ndet, non_blocking=True)
        self._res_h[2].copy_(self.ctl, non_blocking=True)

    def _step(self):
        """enqueue one step (the stage is filled) on the detector's stream behind the caller's stream."""
        cur = torch.cuda.current_stream(self.dev)
        key = self._graph_key()
        with torch.cuda.stream(self.stream):
            self.stream.wait_stream(cur)
            graph = self.graphs.get(key)
            if graph is not None:
                graph.replay()
                self.eng.launches += self._graph_launches
            else:
                l0 = self.eng.launches
                self._enqueue()
                self._warm += 1
                if self._warm >= 2:                                   # buffers exist: capture the step once, replay from now on
                    self._graph_launches = self.eng.launches - l0
                    self.stream.synchronize()
                    saved = self.ctl.clone()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=self.stream):
                        self._enqueue()
                    self.eng.launches -= self._graph_launches          # capture enqueues nothing
                    self.ctl.copy_(saved)                              # (the captured step did not run)
                    self.graphs[key] = g
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._done = ev

    def _dets(self, s: int):
        det_h, ndet_h, _ = self._res_h
        n = int(ndet_h[s])
        d = det_h[s, :n]
        return dict(boxes=d[:, :4].clone(), scores=d[:, 4].clone(), labels=d[:, 5].long())

    def _state(self, s: int):
        self._done.synchronize()
        c = self._res_h[2][RING_CTL * s:RING_CTL * (s + 1)]
        return dict(head=int(c[0]), live=int(c[1]), evicted=int(c[2]), appended=int(c[3]), overflow=bool(c[4]))

    def _live(self, s: int):
        self._done.synchronize()
        torch.cuda.synchronize(self.dev)
        head, n = int(self.ctl[RING_CTL * s]), int(self.ctl[RING_CTL * s + 1])
        idx = s * self.cap + ((head + torch.arange(n, device=self.dev)) & (self.cap - 1))
        return self.pos[idx], self.feat[idx]


class StreamingDetector(_RingDetector):
    """det = StreamingDetector(model, window_us=50_000); det.push(x, y, t, p) -> list with one dict(boxes, scores, labels)."""

    _B, _ring_streams = 1, None

    def __init__(self, model, window_us: int = 50_000, max_chunk: int = 8192, capacity: int = 1 << 17, device=None):
        if model.backbone.use_image:
            raise NotImplementedError("streaming mode drives the events-only model")
        self._setup(model, 1, window_us, max_chunk, capacity, device)
        self.ctl = torch.zeros(RING_CTL, dtype=torch.int32, device=self.dev)

    # ------------------------------------------------------------------------------------------------------------
    def reset(self):
        if self._done is not None:
            self._done.synchronize()
        self.ctl.zero_()

    def _push(self):
        _lib.check(self.lib.dagr_stream_push(_lib.ptr(self.ctl), _lib.ptr(self.stage_d), _lib.ptr(self.batch), _lib.ptr(self.pos),
                                             _lib.ptr(self.feat), self.cap, self.max_chunk, 0, _lib.stream_ptr()), "stream_push")

    def _fill_stage(self, x, y, t, p, t_end):
        n = int(len(t))
        if n > self.max_chunk:
            raise ValueError(f"chunk of {n} events exceeds max_chunk={self.max_chunk}")
        st = self._stage_np
        st[0] = n
        st[1] = int(t_end) - self.window_us
        if n:
            ev = st[4:4 + 4 * n].reshape(n, 4)
            ev[:, 0] = x; ev[:, 1] = y; ev[:, 2] = t; ev[:, 3] = p

    @torch.no_grad()
    def submit(self, x, y, t, p, t_end=None):
        """enqueue one chunk (host arrays: pixel x, y, timestamp t in us (int32 range, non-decreasing across pushes),
        polarity -1/+1).  `t_end` = end of the chunk's time slice (default: its last timestamp); events older than
        t_end - window_us leave the live window.  Returns immediately; `result()` blocks on the step."""
        if self._done is not None:
            self._done.synchronize()                                  # the stage / result buffers of the previous step are free
        if t_end is None:
            t_end = int(t[-1]) if len(t) else int(self._stage_np[1]) + self.window_us
        self._fill_stage(np.asarray(x), np.asarray(y), np.asarray(t), np.asarray(p), t_end)
        self._step()

    def result(self):
        """detections of the last submitted chunk: [dict(boxes f32[n,4] xyxy px, scores f32[n], labels i64[n])] (host tensors)."""
        self._done.synchronize()
        return [self._dets(0)]

    def push(self, x, y, t, p, t_end=None):
        self.submit(x, y, t, p, t_end)
        return self.result()

    @property
    def window_state(self):
        """(head slot, live events, evicted by the last step, appended by the last step, overflow flag) of the last finished step."""
        return self._state(0)

    def live_window(self):
        """(pos int32[n,3], polarity f32[n]) of the live window in arrival order (host sync; for tests)."""
        return self._live(0)


def _check_fusion_model(model, name: str, events_only_class: str):
    if not model.backbone.use_image:
        raise ValueError(f"{name} drives an image-fusion model (backbone.use_image); "
                         f"stream an events-only model with {events_only_class}")
    if model.head.no_events:
        raise NotImplementedError("--no_events: the model has no event path to stream")


class _CameraFrames:
    """The frames of one hybrid camera, for the fusion detectors: two frame slots, the frame pending in the trunk, the frame
    in use, and the done-event of the last step that read each slot.

    set() runs a frame through the model's own ImageBranch (ResNet trunk + CNN head, the captured graphs that model(data)
    replays) on the detector's frame stream and copies its five feature maps and CNN head maps into the slot the steps do
    not use; `slot_dst(slot, feats, outs)` names the destination tensors of a slot (allocating them on first use).  Two
    hazards are ordered on the device: the copy into a slot waits for the last step that read that slot, and the branch's
    static output buffers are overwritten (by the next frame or a model(data) call) only after the copy out of them."""

    def __init__(self, det, slot_dst):
        self.det, self.slot_dst = det, slot_dst
        self.reader = [None, None]            # per slot: done-event of the last step that read it
        self.cur = None                       # slot of the newest usable frame
        self.cur_frame = None                 # (id, t_us) of that frame
        self.pending = None                   # frame whose trunk may still run: dict(slot, id, t_us, ready, trunk)
        self.step_frame = (None, None)        # (id, t_us) of the frame the last submitted step used
        self.nframes = 0
        self.img_h = self.h2d = None

    def check(self, image):
        d = self.det
        if not isinstance(image, torch.Tensor):
            image = torch.from_numpy(np.ascontiguousarray(image))
        if image.dtype != torch.uint8:
            raise ValueError(f"frame dtype {image.dtype}: expected uint8 (raw camera pixels)")
        if image.dim() == 4 and image.shape[0] == 1:
            image = image[0]
        if image.dim() != 3 or tuple(image.shape) != (3, d.H, d.W):
            raise ValueError(f"frame of shape {tuple(image.shape)}: expected [3, {d.H}, {d.W}] or [1, 3, {d.H}, {d.W}]")
        return image.unsqueeze(0)

    def promote(self):
        pend, self.pending = self.pending, None
        self.det.stream.wait_event(pend["ready"])                     # no-op once it completed; orders the very first frame
        self.cur, self.cur_frame = pend["slot"], (pend["id"], pend["t_us"])

    def sync(self):
        if self.pending is not None:
            self.pending["ready"].synchronize()
            self.promote()

    def set(self, image, t_us):
        from .model.image_branch import ImageBranch
        det = self.det
        img = self.check(image)
        self.sync()
        slot = 0 if self.cur is None else 1 - self.cur
        m, fs = det.model, det.frame_stream
        if m._image_branch is None:
            m._image_branch = ImageBranch(m)
        br = m._image_branch
        cur = torch.cuda.current_stream(det.dev)
        if img.is_cuda:
            x = img.to(det.dev).float() / 255.0                        # on the caller's stream, ordered with its writes
        elif self.img_h is None:
            self.img_h = torch.empty(img.shape, dtype=torch.uint8).pin_memory()
        with torch.cuda.stream(fs):
            fs.wait_stream(cur)
            if not img.is_cuda:
                if self.h2d is not None:
                    self.h2d.synchronize()                             # the previous frame's upload has left the pinned stage
                self.img_h.copy_(img)
                x = self.img_h.to(det.dev, non_blocking=True).float() / 255.0    # as format_data
                self.h2d = torch.cuda.Event()
                self.h2d.record(fs)
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(fs)
            feats, outs, (_, ev2) = br.run(x, use_graph=m.image_graph)
            x.record_stream(fs)
            x.record_stream(br.stream)
            fs.wait_event(ev2)
            t1.record(fs)
            if self.reader[slot] is not None:
                fs.wait_event(self.reader[slot])                      # the last step that read this slot is done
            dst_f, dst_o = self.slot_dst(slot, feats, outs)
            for d, s in zip(dst_f, feats):
                d.copy_(s)
            for k, v in outs.items():
                for d, s in zip(dst_o[k], v):
                    d.copy_(s)
            ready = torch.cuda.Event()
            ready.record(fs)
        br.stream.wait_event(ready)                                   # the branch's static outputs outlive the copy
        fid = self.nframes
        self.nframes += 1
        self.pending = dict(slot=slot, id=fid, t_us=t_us, ready=ready, trunk=(t0, t1))
        return fid

    def take_newest(self):
        """before a step: the newest frame whose trunk has finished becomes current (a non-blocking query; the first frame is
        taken whatever its state, the step waits for it on the device).  Returns whether a newer frame is still in flight."""
        if self.pending is not None and (self.cur is None or self.pending["ready"].query()):
            self.promote()
        return self.pending is not None

    def stepped(self, done):
        """after a step was enqueued: it reads the current slot until `done`."""
        self.reader[self.cur] = done
        self.step_frame = self.cur_frame

    def state(self):
        fid, t_us = self.step_frame
        return dict(frame=fid, t_us=t_us, pending=None if self.pending is None else self.pending["id"])


class FusionStreamingDetector(StreamingDetector):
    """Streaming detection with the hybrid (image + events) model: camera frames at frame rate, event chunks in between.

        det = FusionStreamingDetector(model, window_us=50_000)
        fid = det.set_frame(image_u8)          # u8 [3,H,W] or [1,3,H,W], host or device -> frame id 0, 1, 2, ...
        det.push(x, y, t, p)                   # as StreamingDetector: one CUDA graph replay per chunk

    A frame runs through the model's own ImageBranch (ResNet trunk + CNN head, the captured graphs that model(data)
    replays) once, on a side stream, and its five feature maps and CNN head maps are copied into one of two frame slots
    owned by the detector (_CameraFrames).  Each slot has its own captured step graph, so a step is still one replay.

    Which frame a step uses: the newest frame whose trunk has finished when the chunk is submitted (a non-blocking event
    query).  Chunks keep flowing on the previous frame while the next frame's trunk runs; sync_frame() blocks until the
    pending frame is usable, so the next step uses it.  The first step waits for the first frame.  After every step the
    detections equal model(data) over the live window with the image of the frame that frame_state reports."""

    def __init__(self, model, window_us: int = 50_000, max_chunk: int = 8192, capacity: int = 1 << 17, device=None):
        _check_fusion_model(model, "FusionStreamingDetector", "StreamingDetector")
        self._setup(model, 1, window_us, max_chunk, capacity, device)
        self.ctl = torch.zeros(RING_CTL, dtype=torch.int32, device=self.dev)
        self.frame_stream = torch.cuda.Stream(device=self.dev)
        self._slots = None                    # per slot: (image_feats, image_outs) copies of the branch outputs
        self._cam = _CameraFrames(self, self._slot_dst)
        self._overlapped = False              # the last submitted step ran while a newer frame's trunk was in flight

    def _slot_dst(self, slot, feats, outs):
        if self._slots is None:
            self._slots = [([torch.empty_like(f) for f in feats], {k: [torch.empty_like(t) for t in v] for k, v in outs.items()})
                           for _ in range(2)]
        return self._slots[slot]

    @property
    def _cur(self):
        return self._cam.cur

    # ------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def set_frame(self, image, t_us=None):
        """start a new frame: the trunk runs on the device, this returns without waiting for it.  `image` u8 [3,H,W] or
        [1,3,H,W] (host or device); `t_us` is the caller's timestamp of the frame, reported back by frame_state.
        Returns the frame id (0, 1, 2, ...).  A frame still pending is waited for and becomes current first."""
        return self._cam.set(image, t_us)

    def sync_frame(self):
        """block until the pending frame (if any) is usable; the next step uses it."""
        self._cam.sync()

    def _graph_key(self):
        return self._cam.cur

    def _image_inputs(self):
        return self._slots[self._cam.cur]

    @torch.no_grad()
    def submit(self, x, y, t, p, t_end=None):
        """as StreamingDetector.submit; the step uses the newest frame whose trunk has finished (see the class docstring)."""
        self._overlapped = self._cam.take_newest()
        if self._cam.cur is None:
            raise RuntimeError("FusionStreamingDetector: set_frame() must be called before the first chunk")
        super().submit(x, y, t, p, t_end)
        self._cam.stepped(self._done)

    @property
    def frame_state(self):
        """dict(frame=id of the frame the last finished step used, t_us=its timestamp, pending=id of a frame not yet in use
        or None)."""
        if self._done is not None:
            self._done.synchronize()
        return self._cam.state()


def pack_stage(stage: np.ndarray, chunks, t_cut, max_chunk: int, planes=None):
    """write the packed multi-stream stage of dagr_stream_push_multi into the int32 array `stage` (>= 4*S + 4*S*max_chunk
    entries): header [S][4] = {n_new, t_cut, event offset, plane}, then the (x, y, t, polarity) rows of all streams back to
    back.  chunks[s] = (x, y, t, p) host arrays or None (no events).  planes[s] = the frame plane stream s's step reads (image
    fusion, read by the *_planes kernels; the push ignores the word), 0 when `planes` is None.  Returns the per-stream event
    counts."""
    S = len(chunks)
    ns = [0 if c is None else len(c[2]) for c in chunks]
    for s, n in enumerate(ns):
        if n > max_chunk:
            raise ValueError(f"stream {s}: chunk of {n} events exceeds max_chunk={max_chunk}")
    if len(stage) < 4 * S + 4 * S * max_chunk:
        raise ValueError(f"stage of {len(stage)} ints is smaller than 4*S + 4*S*max_chunk = {4 * S + 4 * S * max_chunk}")
    hdr = stage[:4 * S].reshape(S, 4)
    ev = stage[4 * S:4 * S + 4 * S * max_chunk].reshape(S * max_chunk, 4)
    o = 0
    for s, (c, n) in enumerate(zip(chunks, ns)):
        hdr[s] = (n, int(t_cut[s]), o, 0 if planes is None else int(planes[s]))
        if n:
            x, y, t, p = c
            e = ev[o:o + n]
            e[:, 0] = x; e[:, 1] = y; e[:, 2] = t; e[:, 3] = p
        o += n
    return ns


class MultiStreamDetector(_RingDetector):
    """S independent event cameras on one GPU: det = MultiStreamDetector(model, streams=S, window_us=50_000);
    det.push([(x, y, t, p) or None per stream]) -> S dicts(boxes, scores, labels).

    Stream s is sample s of one batched step: its events sit in ring s (`capacity` slots), its window is evicted by its own
    t_cut, and all S windows go through one sort, one event level, one coarse stack and one NMS -- the whole step is one
    CUDA graph replay.  Each stream's detections are those of a StreamingDetector fed the same chunks, and those of the
    synchronous forward over its live window.  All streams share the model (and so its W x H); each keeps its own time base,
    and timestamps only need to be non-decreasing within a stream.  One step advances every stream: a stream with nothing
    new passes None or an empty chunk."""

    def __init__(self, model, streams: int, window_us: int = 50_000, max_chunk: int = 8192, capacity: int = 1 << 17, device=None):
        if model.backbone.use_image:
            raise NotImplementedError("streaming mode drives the events-only model")
        self._setup_streams(model, streams, window_us, max_chunk, capacity, device)

    def _setup_streams(self, model, streams, window_us, max_chunk, capacity, device):
        S = int(streams)
        if not 1 <= S <= MAX_STREAMS:
            raise ValueError(f"streams={streams}: 1 <= streams <= {MAX_STREAMS}")
        cap = _pow2_at_least(capacity)
        if S * cap >= MAX_RING_SLOTS:
            raise ValueError(f"streams * capacity = {S} * {cap} must be < 2^24 (sorted positions are packed in 24 bits)")
        if not 1 <= int(max_chunk) <= cap:
            raise ValueError(f"max_chunk={max_chunk} must be in [1, capacity={cap}]")
        self.S = self._B = self._ring_streams = S
        self._setup(model, S, window_us, max_chunk, cap, device)
        self.ctl = torch.zeros((S + 1) * RING_CTL, dtype=torch.int32, device=self.dev)
        self.stage_bytes = 4 * self.stage_h.numel()

    def _push(self):
        _lib.check(self.lib.dagr_stream_push_multi(_lib.ptr(self.ctl), _lib.ptr(self.stage_d), _lib.ptr(self.batch), _lib.ptr(self.pos),
                                                   _lib.ptr(self.feat), self.cap, self.S, self.max_chunk, _lib.stream_ptr()),
                   "stream_push_multi")

    def reset(self, stream=None):
        """forget the live window of one stream (the others keep theirs) or of all streams."""
        if self._done is not None:
            self._done.synchronize()
        if stream is None:
            self.ctl.zero_()
        else:
            s = int(stream)
            if not 0 <= s < self.S:
                raise IndexError(f"stream {stream} out of range [0, {self.S})")
            self.ctl[RING_CTL * s:RING_CTL * (s + 1)].zero_()

    @torch.no_grad()
    def submit(self, chunks, t_end=None):
        """enqueue one step: chunks[s] = (x, y, t, p) host arrays of stream s (as StreamingDetector.submit) or None.
        t_end[s] = end of stream s's time slice (None, or t_end=None: its last timestamp, or for an empty chunk the previous
        end).  Returns immediately; `result()` blocks on the step."""
        S = self.S
        if len(chunks) != S:
            raise ValueError(f"{len(chunks)} chunks for {S} streams")
        if t_end is not None and len(t_end) != S:
            raise ValueError(f"{len(t_end)} t_end values for {S} streams")
        cs = [None if c is None or len(c[2]) == 0 else tuple(np.asarray(a) for a in c) for c in chunks]
        for s, c in enumerate(cs):
            if c is not None and len(c[2]) > self.max_chunk:
                raise ValueError(f"stream {s}: chunk of {len(c[2])} events exceeds max_chunk={self.max_chunk}")
        if self._done is not None:
            self._done.synchronize()                                  # the stage / result buffers of the previous step are free
        hdr = self._stage_np[:4 * S].reshape(S, 4)
        t_cut = []
        for s, c in enumerate(cs):
            te = None if t_end is None else t_end[s]
            if te is None:
                te = int(c[2][-1]) if c is not None else int(hdr[s, 1]) + self.window_us
            t_cut.append(int(te) - self.window_us)
        pack_stage(self._stage_np, cs, t_cut, self.max_chunk, planes=self._stage_planes())
        self._step()

    def result(self):
        """detections of the last step, one dict(boxes f32[n,4] xyxy px, scores f32[n], labels i64[n]) per stream (host tensors)."""
        self._done.synchronize()
        return [self._dets(s) for s in range(self.S)]

    def push(self, chunks, t_end=None):
        self.submit(chunks, t_end)
        return self.result()

    def window_state(self, s: int):
        """stream s after the last finished step: head slot, live events, evicted / appended by the step, sticky overflow flag."""
        return self._state(s)

    def live_window(self, s: int):
        """(pos int32[n,3], polarity f32[n]) of stream s's live window in arrival order (host sync; for tests)."""
        return self._live(s)

    def _stage_planes(self):
        """word 3 of each stream's stage header: the frame plane of its step (FusionMultiStreamDetector), None for no frames."""
        return None


class FusionMultiStreamDetector(MultiStreamDetector):
    """S hybrid (image + events) cameras on one GPU: MultiStreamDetector with a camera frame per stream.

        det = FusionMultiStreamDetector(model, streams=S, window_us=50_000)
        det.set_frame(s, image_u8)             # per camera, at its own frame rate -> that camera's frame id 0, 1, 2, ...
        det.push([(x, y, t, p) or None per camera], t_end) -> S dicts(boxes, scores, labels)

    Each camera's frames go through the model's own ImageBranch at B = 1, one at a time on the detector's frame stream, and
    their feature maps and CNN head maps are copied into the camera's two frame slots (_CameraFrames, the same bookkeeping as
    FusionStreamingDetector).  Every image tensor the step reads is one plane array [2S, C, h, w]; slot j of camera s is plane
    2s + j.  The plane each camera's step reads travels in word 3 of its stage header, which the step copies to the device
    anyway, and the image kernels read it there (the *_planes entry points): ONE captured step graph serves every
    combination of slots, and the step is one replay.

    Semantics: every camera's image is sampled as a batch of one.  Camera s's detections equal those of a
    FusionStreamingDetector fed the same chunks and frames, and those of model(data) at B = 1 over its live window with the
    frame frame_state(s) reports (the batched model(data) samples with the batch index as a third grid_sample coordinate,
    which is not an exact integer for every sample at every B, so it would tie a camera's bits to the number of cameras).

    Frame policy, per camera: a step uses the camera's newest frame whose copy has finished (a non-blocking event query);
    a camera's first step waits on the device for its first frame; submit raises RuntimeError before any device work while
    some camera has never had a frame.  reset() keeps the frames."""

    def __init__(self, model, streams: int, window_us: int = 50_000, max_chunk: int = 8192, capacity: int = 1 << 17, device=None):
        _check_fusion_model(model, "FusionMultiStreamDetector", "MultiStreamDetector")
        self._setup_streams(model, streams, window_us, max_chunk, capacity, device)
        self.frame_stream = torch.cuda.Stream(device=self.dev)
        self._planes = None                   # (image_feats, image_outs) as plane arrays [2S, ...]
        self._cams = [_CameraFrames(self, lambda j, f, o, s=s: self._plane_dst(2 * s + j, f, o)) for s in range(self.S)]
        self._overlapped = [False] * self.S   # per camera: the last step ran while a newer frame of it was in flight

    def _plane_dst(self, k, feats, outs):
        if self._planes is None:
            n = 2 * self.S
            self._planes = ([torch.empty((n,) + tuple(f.shape[1:]), dtype=f.dtype, device=self.dev) for f in feats],
                            {key: [torch.empty((n,) + tuple(t.shape[1:]), dtype=t.dtype, device=self.dev) for t in v]
                             for key, v in outs.items()})
        pf, po = self._planes
        return [f[k:k + 1] for f in pf], {key: [t[k:k + 1] for t in v] for key, v in po.items()}

    def _camera(self, s):
        s = int(s)
        if not 0 <= s < self.S:
            raise IndexError(f"camera {s} out of range [0, {self.S})")
        return self._cams[s]

    @torch.no_grad()
    def set_frame(self, s: int, image, t_us=None):
        """start a new frame of camera s (see FusionStreamingDetector.set_frame): returns without waiting for the trunk;
        returns camera s's frame id (0, 1, 2, ...).  A frame of camera s still pending is waited for and becomes current."""
        return self._camera(s).set(image, t_us)

    def sync_frame(self, s=None):
        """block until the pending frame of camera s (of every camera when None) is usable; the next step uses it."""
        for c in (self._cams if s is None else [self._camera(s)]):
            c.sync()

    def _image_inputs(self):
        return self._planes

    def _image_planes(self):
        return self.stage_d[3:], 4

    def _stage_planes(self):
        return [2 * s + c.cur for s, c in enumerate(self._cams)]

    @torch.no_grad()
    def submit(self, chunks, t_end=None):
        """as MultiStreamDetector.submit; each camera's step uses its newest frame whose copy has finished."""
        missing = [s for s, c in enumerate(self._cams) if c.cur is None and c.pending is None]
        if missing:
            raise RuntimeError(f"FusionMultiStreamDetector: set_frame() must be called for every camera before the first step "
                               f"(no frame yet: cameras {missing})")
        self._overlapped = [c.take_newest() for c in self._cams]
        super().submit(chunks, t_end)
        for c in self._cams:
            c.stepped(self._done)

    def frame_state(self, s: int):
        """camera s after the last finished step: dict(frame=id of the frame the step used, t_us=its timestamp, pending=id of a
        frame of camera s not yet in use or None)."""
        cam = self._camera(s)
        if self._done is not None:
            self._done.synchronize()
        return cam.state()


def synth_stream(rate_ev_s: int, seconds: float, width: int, height: int, seed: int = 99, kind: str = "uniform"):
    """host arrays (x int16, y int16, t int32 us from 0, p int8) of one continuous synthetic stream."""
    from .data import synth_sample
    n = int(rate_ev_s * seconds)
    window_us = int(seconds * 1e6)
    x, y, t, p = synth_sample(n, width, height, seed, kind, time_window=window_us, window_us=window_us)
    return x.numpy(), y.numpy(), t.numpy(), p.numpy()


def stream_benchmark(dev, size="l", width=640, height=480, rate_ev_s=1_000_000, chunk_us=1000, window_us=50_000, seconds=2.0,
                     kind="uniform", model=None):
    """config 5: per-chunk latency (host submit -> detections on the host) and sustained rate of ONE stream on ONE GPU.
    Latency mode: a chunk is submitted, its detections are awaited, then the next chunk is submitted (a real-time consumer);
    the wall clock per chunk is what a 1 ms chunk period has to accommodate."""
    from .model.dagr import DAGR
    from .utils.args import default_args
    if model is None:
        from tests.helpers import randomize_bn
        torch.manual_seed(0)
        model = randomize_bn(DAGR(default_args(size, batch_size=1), height=height, width=width).eval()).to(dev)
    total_s = seconds + window_us * 1e-6 + 0.02
    x, y, t, p = synth_stream(rate_ev_s, total_s, width, height, kind=kind)
    det = StreamingDetector(model, window_us=window_us, max_chunk=max(4096, int(rate_ev_s * chunk_us * 1e-6 * 4)))
    bounds = np.searchsorted(t, np.arange(0, int(total_s * 1e6) + chunk_us, chunk_us))
    nchunks = len(bounds) - 1
    lat, dev_ms, evs = [], [], []
    warm = int(window_us / chunk_us) + 20                                # fill the live window first (+ graph capture)
    import gc
    gc_was = gc.isenabled()
    gc.collect()
    gc.disable()                                                         # a collector pause inside a 1 ms chunk period is a latency spike
    for k in range(nchunks):
        a, b = int(bounds[k]), int(bounds[k + 1])
        t_end = (k + 1) * chunk_us
        if k >= warm:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(det.stream)
            det.submit(x[a:b], y[a:b], t[a:b], p[a:b], t_end)
            e1.record(det.stream)
            out = det.result()
            lat.append((time.perf_counter() - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            evs.append(b - a)
        else:
            det.push(x[a:b], y[a:b], t[a:b], p[a:b], t_end)
    if gc_was:
        gc.enable()
    st = det.window_state
    lat_s, dev_s = sorted(lat), sorted(dev_ms)
    q = lambda v, f: v[min(len(v) - 1, int(f * len(v)))]
    busy = sum(lat) * 1e-3
    return dict(model=f"dagr-{size}", stream_rate_mev_s=rate_ev_s / 1e6, chunk_us=chunk_us, window_us=window_us,
                stream_seconds=len(lat) * chunk_us * 1e-6, chunks=len(lat), events_per_chunk=float(np.mean(evs)),
                live_events=st["live"], overflow=st["overflow"],
                latency_ms=dict(p50=q(lat_s, 0.5), p90=q(lat_s, 0.9), p99=q(lat_s, 0.99), max=lat_s[-1]),
                device_ms=dict(p50=q(dev_s, 0.5), p99=q(dev_s, 0.99)),
                sustained_mev_s=sum(evs) / busy / 1e6, realtime=bool(q(lat_s, 0.99) * 1e3 <= chunk_us),
                realtime_margin=chunk_us / (q(lat_s, 0.5) * 1e3),
                note="one stream on one GPU; every chunk: H2D of the chunk from pinned memory, eviction by watermark + append into the "
                     "device ring, full forward over the live window, NMS, D2H of the detections -- one CUDA graph replay; latency = host "
                     "wall clock from submit() to the detections being readable on the host, chunks submitted back to back "
                     "(sustained_mev_s = events / busy time: how much faster than the 1 Mevents/s feed the loop runs); Python's cyclic garbage "
                     "collector is paused during the timed loop")


def multistream_benchmark(dev, streams, size="l", width=640, height=480, rate_ev_s=1_000_000, chunk_us=1000, window_us=50_000,
                          seconds=2.0, kind="uniform", model=None, capacity=1 << 17):
    """config 5 with S cameras on ONE GPU: S independent synthetic streams (seeds 99, 100, ...) at `rate_ev_s` each, all
    advanced by one MultiStreamDetector step per chunk period.  Latency mode as in stream_benchmark: a step is submitted,
    the detections of all S streams are awaited on the host, then the next step is submitted."""
    from .model.dagr import DAGR
    from .utils.args import default_args
    S = int(streams)
    if model is None:
        from tests.helpers import randomize_bn
        torch.manual_seed(0)
        model = randomize_bn(DAGR(default_args(size, batch_size=1), height=height, width=width).eval()).to(dev)
    total_s = seconds + window_us * 1e-6 + 0.02
    evs_s = [synth_stream(rate_ev_s, total_s, width, height, seed=99 + s, kind=kind) for s in range(S)]
    det = MultiStreamDetector(model, streams=S, window_us=window_us, max_chunk=max(4096, int(rate_ev_s * chunk_us * 1e-6 * 4)),
                              capacity=capacity)
    grid = np.arange(0, int(total_s * 1e6) + chunk_us, chunk_us)
    bounds = [np.searchsorted(e[2], grid) for e in evs_s]
    nchunks = len(grid) - 1
    lat, dev_ms, evs = [], [], []
    warm = int(window_us / chunk_us) + 20                                # fill the live windows first (+ graph capture)
    import gc
    gc_was = gc.isenabled()
    gc.collect()
    gc.disable()                                                         # a collector pause inside a 1 ms chunk period is a latency spike
    for k in range(nchunks):
        chunks = []
        for (x, y, t, p), bd in zip(evs_s, bounds):
            a, b = int(bd[k]), int(bd[k + 1])
            chunks.append((x[a:b], y[a:b], t[a:b], p[a:b]))
        t_end = [(k + 1) * chunk_us] * S
        if k >= warm:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(det.stream)
            det.submit(chunks, t_end)
            e1.record(det.stream)
            det.result()
            lat.append((time.perf_counter() - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            evs.append(sum(len(c[2]) for c in chunks))
        else:
            det.push(chunks, t_end)
    if gc_was:
        gc.enable()
    st = [det.window_state(s) for s in range(S)]
    lat_s, dev_s = sorted(lat), sorted(dev_ms)
    q = lambda v, f: v[min(len(v) - 1, int(f * len(v)))]
    busy = sum(lat) * 1e-3
    return dict(model=f"dagr-{size}", streams=S, kind=kind, stream_rate_mev_s=rate_ev_s / 1e6, chunk_us=chunk_us, window_us=window_us,
                stream_seconds=len(lat) * chunk_us * 1e-6, steps=len(lat), events_per_step=float(np.mean(evs)),
                stage_bytes=det.stage_bytes, live_events=[x["live"] for x in st], overflow=[x["overflow"] for x in st],
                latency_ms=dict(p50=q(lat_s, 0.5), p90=q(lat_s, 0.9), p99=q(lat_s, 0.99), max=lat_s[-1]),
                device_ms=dict(p50=q(dev_s, 0.5), p99=q(dev_s, 0.99)),
                sustained_mev_s=sum(evs) / busy / 1e6, realtime=bool(q(lat_s, 0.99) * 1e3 <= chunk_us),
                realtime_margin=chunk_us / (q(lat_s, 0.5) * 1e3),
                note=f"{S} independent streams on one GPU, one MultiStreamDetector step per chunk period: H2D of the packed stage "
                     "(fixed size), per-stream eviction + append into S device rings, one batched forward over the S live windows, "
                     "NMS, D2H of the detections -- one CUDA graph replay; latency = host wall clock from submit() until the "
                     "detections of all streams are readable on the host; sustained_mev_s = events of all streams / busy time; "
                     "Python's cyclic garbage collector is paused during the timed loop")


def fusion_stream_benchmark(dev, size="s", img_net="resnet50", width=640, height=480, rate_ev_s=1_000_000, chunk_us=1000,
                            window_us=50_000, seconds=2.0, frame_us=50_000, sync_frames=False, kind="uniform", model=None,
                            step_priority=0):
    """config 3's hybrid model on config 5's stream: one event stream in `chunk_us` chunks and a new camera frame every
    `frame_us` of stream time, through FusionStreamingDetector.  Latency mode as in stream_benchmark (a chunk is submitted,
    its detections are awaited, then the next one); frames are set between two chunks, followed by sync_frame() when
    `sync_frames`.  Frames are seeded random u8 images on the host (the trunk's cost does not depend on the pixels).
    step_priority < 0 runs the steps on a higher-priority stream than the trunk's (an experiment: does it shield the chunks?)."""
    from .model.dagr import DAGR
    from .utils.args import default_args
    if model is None:
        from tests.helpers import randomize_bn
        torch.manual_seed(0)
        model = randomize_bn(DAGR(default_args(size, batch_size=1, use_image=True, img_net=img_net), height=height, width=width).eval()).to(dev)
    total_s = seconds + window_us * 1e-6 + 0.02
    x, y, t, p = synth_stream(rate_ev_s, total_s, width, height, kind=kind)
    g = torch.Generator().manual_seed(0)
    frames = [torch.randint(0, 256, (3, height, width), generator=g, dtype=torch.uint8) for _ in range(4)]
    det = FusionStreamingDetector(model, window_us=window_us, max_chunk=max(4096, int(rate_ev_s * chunk_us * 1e-6 * 4)))
    if step_priority:
        det.stream = torch.cuda.Stream(device=det.dev, priority=step_priority)      # before the first step: captures inherit it
    bounds = np.searchsorted(t, np.arange(0, int(total_s * 1e6) + chunk_us, chunk_us))
    nchunks = len(bounds) - 1
    lat, dev_ms, evs, overlapped, set_ms, trunk, first_use = [], [], [], [], [], [], []
    waiting = {}                                                         # frame id -> host time of its set_frame
    warm = int(window_us / chunk_us) + 20                                # fill the live window first (+ both graph captures)
    import gc
    gc_was = gc.isenabled()
    gc.collect()
    gc.disable()                                                         # a collector pause inside a 1 ms chunk period is a latency spike
    for k in range(nchunks):
        a, b = int(bounds[k]), int(bounds[k + 1])
        t_end = (k + 1) * chunk_us
        if (k * chunk_us) % frame_us == 0:                              # the camera delivers a frame at stream time k * chunk_us
            ts = time.perf_counter()
            fid = det.set_frame(frames[(k * chunk_us // frame_us) % len(frames)], t_us=k * chunk_us)
            tr = det._cam.pending["trunk"]
            if sync_frames:
                det.sync_frame()
            if k >= warm:
                set_ms.append((time.perf_counter() - ts) * 1e3)
                trunk.append(tr)
                waiting[fid] = ts
        if k >= warm:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(det.stream)
            det.submit(x[a:b], y[a:b], t[a:b], p[a:b], t_end)
            e1.record(det.stream)
            det.result()
            t1 = time.perf_counter()
            lat.append((t1 - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            evs.append(b - a)
            overlapped.append(det._overlapped)
            fid = det._cam.step_frame[0]
            if fid in waiting:
                first_use.append((t1 - waiting.pop(fid)) * 1e3)
        else:
            det.push(x[a:b], y[a:b], t[a:b], p[a:b], t_end)
    if gc_was:
        gc.enable()
    torch.cuda.synchronize(dev)
    trunk_ms = [a.elapsed_time(b) for a, b in trunk]
    st = det.window_state
    q = lambda v, f: v[min(len(v) - 1, int(f * len(v)))]

    def dist(v):
        v = sorted(v)
        return dict(n=len(v), p50=q(v, 0.5), p99=q(v, 0.99), max=v[-1]) if v else dict(n=0)

    busy = sum(lat) * 1e-3
    return dict(model=f"dagr-{size} + {img_net}", width=width, height=height, stream_rate_mev_s=rate_ev_s / 1e6, chunk_us=chunk_us,
                window_us=window_us, frame_us=frame_us, sync_frames=bool(sync_frames), step_priority=step_priority, stream_seconds=len(lat) * chunk_us * 1e-6,
                chunks=len(lat), frames=len(trunk_ms), events_per_chunk=float(np.mean(evs)), live_events=st["live"], overflow=st["overflow"],
                latency_ms=dist(lat), latency_ms_trunk_in_flight=dist([v for v, o in zip(lat, overlapped) if o]),
                latency_ms_no_trunk=dist([v for v, o in zip(lat, overlapped) if not o]),
                device_ms=dist(dev_ms), trunk_device_ms=dist(trunk_ms), set_frame_host_ms=dist(set_ms),
                frame_to_first_use_ms=dist(first_use), sustained_mev_s=sum(evs) / busy / 1e6,
                note="one hybrid stream on one GPU: every chunk is one CUDA graph replay of the step of the current frame slot; every "
                     "frame_us of stream time a host u8 frame goes through the ResNet trunk + CNN head (captured ImageBranch graphs) on "
                     "a side stream and is copied into the free slot.  latency = host wall clock from submit() to the detections on the "
                     "host; *_trunk_in_flight = chunks submitted while a newer frame's trunk had not finished (they use the previous "
                     "frame); device_ms = CUDA events around the step on the detector's stream; trunk_device_ms = CUDA events around "
                     "the branch on the frame stream; set_frame_host_ms = host time of set_frame (+ sync_frame when sync_frames); "
                     "frame_to_first_use_ms = host time from set_frame until the detections of the first step using that frame are on "
                     "the host; chunks are submitted back to back, faster than the real 1 ms period, so frames arrive every "
                     "frame_us / chunk_us chunks rather than every frame_us of wall time; Python's cyclic garbage collector is paused "
                     "during the timed loop")


def fusion_multistream_benchmark(dev, streams, size="s", img_net="resnet50", width=640, height=480, rate_ev_s=1_000_000,
                                 chunk_us=1000, window_us=50_000, seconds=2.0, frame_us=50_000, kind="uniform", model=None,
                                 capacity=1 << 17):
    """S hybrid cameras on ONE GPU through FusionMultiStreamDetector: S independent synthetic event streams (seeds 99, 100,
    ...) at `rate_ev_s` each, advanced by one step per chunk period, and a new frame every `frame_us` of stream time per
    camera, camera s's frames offset by s * frame_us / S (rounded down to the chunk grid) so that the trunks spread out.
    Latency mode as in multistream_benchmark: a step is submitted, the detections of all S cameras are awaited, then the next
    step is submitted; frames are set between two steps and never waited for."""
    from .model.dagr import DAGR
    from .utils.args import default_args
    S = int(streams)
    if model is None:
        from tests.helpers import randomize_bn
        torch.manual_seed(0)
        model = randomize_bn(DAGR(default_args(size, batch_size=1, use_image=True, img_net=img_net), height=height, width=width).eval()).to(dev)
    total_s = seconds + window_us * 1e-6 + 0.02
    evs_s = [synth_stream(rate_ev_s, total_s, width, height, seed=99 + s, kind=kind) for s in range(S)]
    g = torch.Generator().manual_seed(0)
    frames = [torch.randint(0, 256, (3, height, width), generator=g, dtype=torch.uint8) for _ in range(4)]
    det = FusionMultiStreamDetector(model, streams=S, window_us=window_us, max_chunk=max(4096, int(rate_ev_s * chunk_us * 1e-6 * 4)),
                                    capacity=capacity)
    offset = [(s * frame_us // S) // chunk_us * chunk_us for s in range(S)]
    grid = np.arange(0, int(total_s * 1e6) + chunk_us, chunk_us)
    bounds = [np.searchsorted(e[2], grid) for e in evs_s]
    nchunks = len(grid) - 1
    lat, dev_ms, evs, overlapped, trunk = [], [], [], [], []
    first_use = [[] for _ in range(S)]
    waiting = {}                                                         # (camera, frame id) -> host time of its set_frame
    warm = int(window_us / chunk_us) + 20                                # fill the live windows first (+ graph capture)
    for s in range(S):                                                   # every camera needs a frame before the first step
        det.set_frame(s, frames[s % len(frames)], t_us=0)
    import gc
    gc_was = gc.isenabled()
    gc.collect()
    gc.disable()                                                         # a collector pause inside a 1 ms chunk period is a latency spike
    for k in range(nchunks):
        tk = k * chunk_us
        for s in range(S):
            if tk > offset[s] and (tk - offset[s]) % frame_us == 0:      # camera s delivers a frame at stream time tk
                ts = time.perf_counter()
                fid = det.set_frame(s, frames[(s + (tk - offset[s]) // frame_us) % len(frames)], t_us=tk)
                if k >= warm:
                    trunk.append(det._cams[s].pending["trunk"])
                    waiting[(s, fid)] = ts
        chunks = []
        for (x, y, t, p), bd in zip(evs_s, bounds):
            a, b = int(bd[k]), int(bd[k + 1])
            chunks.append((x[a:b], y[a:b], t[a:b], p[a:b]))
        t_end = [(k + 1) * chunk_us] * S
        if k >= warm:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(det.stream)
            det.submit(chunks, t_end)
            e1.record(det.stream)
            det.result()
            t1 = time.perf_counter()
            lat.append((t1 - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            evs.append(sum(len(c[2]) for c in chunks))
            overlapped.append(any(det._overlapped))
            for s, cam in enumerate(det._cams):
                key = (s, cam.step_frame[0])
                if key in waiting:
                    first_use[s].append((t1 - waiting.pop(key)) * 1e3)
        else:
            det.push(chunks, t_end)
    if gc_was:
        gc.enable()
    torch.cuda.synchronize(dev)
    trunk_ms = [a.elapsed_time(b) for a, b in trunk]
    st = [det.window_state(s) for s in range(S)]
    q = lambda v, f: v[min(len(v) - 1, int(f * len(v)))]

    def dist(v):
        v = sorted(v)
        return dict(n=len(v), p50=q(v, 0.5), p99=q(v, 0.99), max=v[-1]) if v else dict(n=0)

    busy = sum(lat) * 1e-3
    return dict(model=f"dagr-{size} + {img_net}", streams=S, width=width, height=height, stream_rate_mev_s=rate_ev_s / 1e6,
                chunk_us=chunk_us, window_us=window_us, frame_us=frame_us, frame_offset_us=offset, stream_seconds=len(lat) * chunk_us * 1e-6,
                steps=len(lat), frames=len(trunk_ms), events_per_step=float(np.mean(evs)), live_events=[x["live"] for x in st],
                overflow=[x["overflow"] for x in st], graphs=len(det.graphs), latency_ms=dist(lat),
                latency_ms_trunk_in_flight=dist([v for v, o in zip(lat, overlapped) if o]),
                latency_ms_no_trunk=dist([v for v, o in zip(lat, overlapped) if not o]), steps_trunk_in_flight=int(sum(overlapped)),
                device_ms=dist(dev_ms), trunk_device_ms=dist(trunk_ms), frame_to_first_use_ms=[dist(v) for v in first_use],
                sustained_mev_s=sum(evs) / busy / 1e6,
                note=f"{S} hybrid cameras on one GPU, one FusionMultiStreamDetector step (one CUDA graph replay) per chunk period; every "
                     "frame_us of stream time each camera's host u8 frame goes through the ResNet trunk + CNN head at B = 1 (captured "
                     "ImageBranch graphs) on the frame stream and is copied into the camera's free plane; latency = host wall clock "
                     "from submit() until the detections of all cameras are on the host; *_trunk_in_flight = steps submitted while "
                     "some camera's newer frame had not finished; device_ms = CUDA events around the step on the detector's stream; "
                     "trunk_device_ms = CUDA events around the branch on the frame stream; frame_to_first_use_ms[s] = host time from "
                     "set_frame of camera s until the detections of the first step using that frame are on the host; steps are "
                     "submitted back to back, faster than the real 1 ms period, so frames arrive every frame_us / chunk_us steps "
                     "rather than every frame_us of wall time; Python's cyclic garbage collector is paused during the timed loop")
