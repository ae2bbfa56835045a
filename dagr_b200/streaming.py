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
                                 ring=self.ctl, ring_streams=self._ring_streams)
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


class FusionStreamingDetector(StreamingDetector):
    """Streaming detection with the hybrid (image + events) model: camera frames at frame rate, event chunks in between.

        det = FusionStreamingDetector(model, window_us=50_000)
        fid = det.set_frame(image_u8)          # u8 [3,H,W] or [1,3,H,W], host or device -> frame id 0, 1, 2, ...
        det.push(x, y, t, p)                   # as StreamingDetector: one CUDA graph replay per chunk

    A frame runs through the model's own ImageBranch (ResNet trunk + CNN head, the captured graphs that model(data)
    replays) once, on the branch's side stream, and its five feature maps and CNN head maps are copied into one of two frame
    slots owned by the detector.  Each slot has its own captured step graph, so a step is still one replay.

    Which frame a step uses: the newest frame whose trunk has finished when the chunk is submitted (a non-blocking event
    query).  Chunks keep flowing on the previous frame while the next frame's trunk runs; sync_frame() blocks until the
    pending frame is usable, so the next step uses it.  The first step waits for the first frame.  After every step the
    detections equal model(data) over the live window with the image of the frame that frame_state reports.

    Two hazards are ordered on the device: a slot is overwritten only after the last step that read it (the copy waits for
    that step), and the branch's static output buffers are overwritten (by the next frame or a model(data) call) only after
    the copy out of them (the branch stream waits for the copy)."""

    def __init__(self, model, window_us: int = 50_000, max_chunk: int = 8192, capacity: int = 1 << 17, device=None):
        if not model.backbone.use_image:
            raise ValueError("FusionStreamingDetector drives an image-fusion model (backbone.use_image); "
                             "stream an events-only model with StreamingDetector")
        if model.head.no_events:
            raise NotImplementedError("--no_events: the model has no event path to stream")
        self._setup(model, 1, window_us, max_chunk, capacity, device)
        self.ctl = torch.zeros(RING_CTL, dtype=torch.int32, device=self.dev)
        self.frame_stream = torch.cuda.Stream(device=self.dev)
        self._slots = None                    # per slot: (image_feats, image_outs) copies of the branch outputs
        self._reader = [None, None]           # per slot: done-event of the last step that read it
        self._cur = None                      # slot of the newest usable frame
        self._cur_frame = None                # (id, t_us) of that frame
        self._pending = None                  # frame whose trunk may still run: dict(slot, id, t_us, ready, trunk)
        self._step_frame = (None, None)       # (id, t_us) of the frame the last submitted step used
        self._overlapped = False              # the last submitted step ran while a newer frame's trunk was in flight
        self._nframes = 0
        self._img_h = self._h2d = None

    # ------------------------------------------------------------------------------------------------------------
    def _check_frame(self, image):
        if not isinstance(image, torch.Tensor):
            image = torch.from_numpy(np.ascontiguousarray(image))
        if image.dtype != torch.uint8:
            raise ValueError(f"frame dtype {image.dtype}: expected uint8 (raw camera pixels)")
        if image.dim() == 4 and image.shape[0] == 1:
            image = image[0]
        if image.dim() != 3 or tuple(image.shape) != (3, self.H, self.W):
            raise ValueError(f"frame of shape {tuple(image.shape)}: expected [3, {self.H}, {self.W}] or [1, 3, {self.H}, {self.W}]")
        return image.unsqueeze(0)

    def _promote(self):
        pend, self._pending = self._pending, None
        self.stream.wait_event(pend["ready"])                         # no-op once it completed; orders the very first frame
        self._cur, self._cur_frame = pend["slot"], (pend["id"], pend["t_us"])

    @torch.no_grad()
    def set_frame(self, image, t_us=None):
        """start a new frame: the trunk runs on the device, this returns without waiting for it.  `image` u8 [3,H,W] or
        [1,3,H,W] (host or device); `t_us` is the caller's timestamp of the frame, reported back by frame_state.
        Returns the frame id (0, 1, 2, ...).  A frame still pending is waited for and becomes current first."""
        from .model.image_branch import ImageBranch
        img = self._check_frame(image)
        self.sync_frame()
        slot = 0 if self._cur is None else 1 - self._cur
        m, fs = self.model, self.frame_stream
        if m._image_branch is None:
            m._image_branch = ImageBranch(m)
        br = m._image_branch
        cur = torch.cuda.current_stream(self.dev)
        if img.is_cuda:
            x = img.to(self.dev).float() / 255.0                       # on the caller's stream, ordered with its writes
        elif self._img_h is None:
            self._img_h = torch.empty(img.shape, dtype=torch.uint8).pin_memory()
        with torch.cuda.stream(fs):
            fs.wait_stream(cur)
            if not img.is_cuda:
                if self._h2d is not None:
                    self._h2d.synchronize()                            # the previous frame's upload has left the pinned stage
                self._img_h.copy_(img)
                x = self._img_h.to(self.dev, non_blocking=True).float() / 255.0   # as format_data
                self._h2d = torch.cuda.Event()
                self._h2d.record(fs)
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(fs)
            feats, outs, (_, ev2) = br.run(x, use_graph=m.image_graph)
            x.record_stream(fs)
            x.record_stream(br.stream)
            fs.wait_event(ev2)
            t1.record(fs)
            if self._slots is None:
                self._slots = [([torch.empty_like(f) for f in feats], {k: [torch.empty_like(t) for t in v] for k, v in outs.items()})
                               for _ in range(2)]
            if self._reader[slot] is not None:
                fs.wait_event(self._reader[slot])                     # the last step that read this slot is done
            dst_f, dst_o = self._slots[slot]
            for d, s in zip(dst_f, feats):
                d.copy_(s)
            for k, v in outs.items():
                for d, s in zip(dst_o[k], v):
                    d.copy_(s)
            ready = torch.cuda.Event()
            ready.record(fs)
        br.stream.wait_event(ready)                                   # the branch's static outputs outlive the copy
        fid = self._nframes
        self._nframes += 1
        self._pending = dict(slot=slot, id=fid, t_us=t_us, ready=ready, trunk=(t0, t1))
        return fid

    def sync_frame(self):
        """block until the pending frame (if any) is usable; the next step uses it."""
        if self._pending is not None:
            self._pending["ready"].synchronize()
            self._promote()

    def _graph_key(self):
        return self._cur

    def _image_inputs(self):
        return self._slots[self._cur]

    @torch.no_grad()
    def submit(self, x, y, t, p, t_end=None):
        """as StreamingDetector.submit; the step uses the newest frame whose trunk has finished (see the class docstring)."""
        if self._pending is not None and (self._cur is None or self._pending["ready"].query()):
            self._promote()
        if self._cur is None:
            raise RuntimeError("FusionStreamingDetector: set_frame() must be called before the first chunk")
        self._overlapped = self._pending is not None
        super().submit(x, y, t, p, t_end)
        self._reader[self._cur] = self._done
        self._step_frame = self._cur_frame

    @property
    def frame_state(self):
        """dict(frame=id of the frame the last finished step used, t_us=its timestamp, pending=id of a frame not yet in use
        or None)."""
        if self._done is not None:
            self._done.synchronize()
        fid, t_us = self._step_frame
        return dict(frame=fid, t_us=t_us, pending=None if self._pending is None else self._pending["id"])


def pack_stage(stage: np.ndarray, chunks, t_cut, max_chunk: int):
    """write the packed multi-stream stage of dagr_stream_push_multi into the int32 array `stage` (>= 4*S + 4*S*max_chunk
    entries): header [S][4] = {n_new, t_cut, event offset, 0}, then the (x, y, t, polarity) rows of all streams back to back.
    chunks[s] = (x, y, t, p) host arrays or None (no events).  Returns the per-stream event counts."""
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
        hdr[s] = (n, int(t_cut[s]), o, 0)
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
        pack_stage(self._stage_np, cs, t_cut, self.max_chunk)
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
            tr = det._pending["trunk"]
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
            fid = det._step_frame[0]
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
