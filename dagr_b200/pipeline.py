"""Host -> device input pipeline: the next batch's H2D copy runs on a side stream while the current batch is
processed (the reference copies synchronously inside the loop: utils/testing.py:29)."""
from __future__ import annotations

import torch


class Prefetcher:
    """iterates over pinned host batches; `next()` returns a device batch whose copy was enqueued one step earlier."""

    def __init__(self, batches, device, transform=None):
        self.batches, self.device, self.transform = list(batches), device, transform
        self.stream = torch.cuda.Stream(device=device)
        self._next = None
        self._i = 0

    def _issue(self, i):
        with torch.cuda.stream(self.stream):
            d = self.batches[i % len(self.batches)].to(self.device, non_blocking=True)
            if self.transform is not None:
                d = self.transform(d)
        ev = torch.cuda.Event()
        ev.record(self.stream)
        return d, ev

    def next(self):
        if self._next is None:
            self._next = self._issue(self._i)
        d, ev = self._next
        self._i += 1
        self._next = self._issue(self._i)                   # overlaps with the caller's compute on `d`
        torch.cuda.current_stream().wait_event(ev)
        for v in d.__dict__.values():                       # tensors were allocated on the side stream
            if torch.is_tensor(v) and v.is_cuda:
                v.record_stream(torch.cuda.current_stream())
        return d


class PipelinedDetector:
    """Throughput-oriented front end of `DAGR.forward` for independent batches (reset=True forwards).

        det = PipelinedDetector(model)
        h = det.submit(batch0)
        for batch in batches[1:]:
            h_next = det.submit(batch)        # enqueue step i+1 ...
            detections = h.result()           # ... before blocking on step i
            h = h_next

    `submit` enqueues the event-level kernels on the caller's stream and the coarse stack + NMS + the device->host
    copy of the detections on the engine's side stream (`Engine.overlap`), so consecutive steps overlap on the GPU and the
    host never waits inside `submit`.  `result()` blocks on that step's event and returns the same list of dicts
    (`boxes`, `scores`, `labels`) as `DAGR.forward(...)[0]` (src/dagr/model/utils.py:104-108), as host tensors.
    At most two steps may be in flight (results live in two alternating pinned buffers).

    Image-fusion models (--use_image) take `data.image` as `model(data)` does (the loader's u8 frames or formatted
    floats, in the model's image_precision).  Their forwards run on a stream of the detector that waits for the caller's
    stream as of `submit`, and the image branch of step i+1 waits only for that point and for step i-1, the last reader
    of the branch outputs of its hand-off slot (ImageBranch.run(slot=...)): it runs next to the event-level kernels, the
    coarse stack and the NMS of step i.  The coarse stack with its image sampling replays as one CUDA graph per slot.
    The caller's stream waits for the points where the batch has been read.  The detections are those of `model(data)`
    on the same batch, bit for bit.  --no_events models have no event path to pipeline and are refused.
    """

    class Handle:
        def __init__(self, event, det_h, ndet_h):
            self.event, self.det_h, self.ndet_h = event, det_h, ndet_h

        def result(self):
            self.event.synchronize()
            out = []
            for b, n in enumerate(self.ndet_h.tolist()):
                d = self.det_h[b, :n]
                out.append(dict(boxes=d[:, :4].clone(), scores=d[:, 4].clone(), labels=d[:, 5].long()))
            return out

    def __init__(self, model):
        self.model = model
        self.engine = model.engine
        self._host = {}
        self._k = 0
        self._stream = None                  # image fusion: the stream the forwards run on

    def _check(self, data):
        """the argument checks of submit(), before any device work."""
        m = self.model
        if not m.backbone.use_image:
            return
        if m.head.no_events:
            raise ValueError("PipelinedDetector pipelines the event path; a --no_events model has none (use model(data))")
        img = getattr(data, "image", None)
        if not torch.is_tensor(img):
            raise ValueError("an image-fusion model needs data.image: u8 or float frames [B, 3, H, W]")
        if img.dim() != 4 or img.shape[1] != 3 or not (img.dtype == torch.uint8 or img.dtype.is_floating_point):
            raise ValueError(f"data.image {tuple(img.shape)} {img.dtype}: expected u8 or float frames [B, 3, H, W]")
        B = int(getattr(data, "num_graphs", 0) or 0)
        if B and int(img.shape[0]) != B:
            raise ValueError(f"data.image holds {int(img.shape[0])} frames for a batch of {B} samples")
        if img.device != data.pos.device:
            raise ValueError(f"data.image is on {img.device}, the events on {data.pos.device}")
        if m.keep_stream:
            raise ValueError("PipelinedDetector runs reset=True forwards of independent batches; keep_stream=True starts an "
                             "incremental stream (use model(data) or AsyncDAGR)")

    def submit(self, data, filtering=True) -> "PipelinedDetector.Handle":
        self._check(data)
        if not self.model.backbone.use_image:
            return self._step(data, filtering)
        # image fusion: the forward runs on a stream of the detector, so that the caller's stream holds nothing of it.  The
        # image branch then waits for the caller's stream as of this call (where the batch is valid) and for the last reader
        # of its slot, not for the event-level kernels of the batch before; the caller's stream waits for the points where
        # the batch has been read, so it may write the batch's tensors again, as after a synchronous call
        cur = torch.cuda.current_stream(data.pos.device)
        if self._stream is None:
            self._stream = torch.cuda.Stream(device=data.pos.device)
        ready = torch.cuda.Event()
        ready.record(cur)
        self._stream.wait_event(ready)
        read = []
        with torch.cuda.stream(self._stream):
            h = self._step(data, filtering, frame_ready=ready, inputs_read=read)
        for v in data.__dict__.values():                    # read on the detector's stream, which the caller never waits for
            if torch.is_tensor(v) and v.is_cuda:
                v.record_stream(self._stream)
        for ev in read:
            cur.wait_event(ev)
        return h

    def _step(self, data, filtering, **kw) -> "PipelinedDetector.Handle":
        m, eng = self.model, self.engine
        prev = eng.overlap
        eng.overlap = True
        try:
            dec = m.forward_decoded(data, reset=True, **kw)
            det, ndet = eng.postprocess(dec, m.conf_threshold, m.nms_threshold, m.width, m.height, filtering=filtering)
            k = self._k & 1
            self._k += 1
            key = (k, tuple(det.shape))
            if key not in self._host:
                self._host[key] = (torch.empty(det.shape, dtype=det.dtype).pin_memory(),
                                   torch.empty(ndet.shape, dtype=ndet.dtype).pin_memory())
            det_h, ndet_h = self._host[key]
            with eng.result_stream():
                det_h.copy_(det, non_blocking=True)
                ndet_h.copy_(ndet, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
            eng.fence()                                                  # the slot is free once its results left the device
        finally:
            eng.overlap = prev
        return PipelinedDetector.Handle(ev, det_h, ndet_h)
