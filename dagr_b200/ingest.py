"""Event ingest on the device: raw DSEC events -> the int32 arrays the graph builder eats (SURVEY 8(f) rank 1).

Host-side mirror of the reference's CPU functions for this step, same names and argument meaning:

  downsample_events(events, input_height, input_width, output_height, output_width, change_map=None)
      scripts/downsample_events.py:91-106 -- dict of CUDA tensors instead of numpy arrays, the change map is a CUDA
      tensor carried from chunk to chunk exactly like the script's main loop does (:146-153)
  ingest_window(events, width, height, time_window, t_cut=None, sample=0)
      dsec_data.py:141-147,177-179 + data/utils.py:6-20 + utils/buffers.py:33-44 + ev_tgn.py:11-16 fused
  collate(samples, width, height, time_window)
      the duck-typed Batch `DAGR.forward` accepts (pos_denorm shortcut, ev_tgn.py:12-13)
  preprocess_image(frames_u8, height, width, scale)
      dsec_data.py:149-154 -- crop, cv2.resize(INTER_CUBIC) by an integer factor and HWC -> CHW, bit for bit

Everything runs in hand-written kernels (csrc/ingest.cu) on the current stream; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from .data import EventBatch


def _i32(n, dev):
    return torch.empty(max(int(n), 1), dtype=torch.int32, device=dev)


def _as(t: torch.Tensor, dtype, name):
    _lib.require_cuda(t, name)
    if t.dtype != dtype:
        t = t.to(dtype)
    return t.contiguous()


def _xy16(t, name):
    # uint16 coordinates (h5 dtype of the DSEC files); torch.uint16 and int16 share the bit pattern for 0..32767
    _lib.require_cuda(t, name)
    if t.dtype in (torch.uint16, torch.int16):
        return t.contiguous()
    return t.to(torch.int16).contiguous()


def downsample_events(events: Dict[str, torch.Tensor], input_height: int, input_width: int, output_height: int,
                      output_width: int, change_map: Optional[torch.Tensor] = None):
    """events: x, y (u16/int16), p (int8, +-1), t (int64), time-ordered, on CUDA.  Returns (events at the output
    resolution, change_map float32[output_height, output_width])."""
    lib = _lib.load()
    x, y = _xy16(events["x"], "x"), _xy16(events["y"], "y")
    p = _as(events["p"].reshape(-1), torch.int8, "p")
    t = _as(events["t"].reshape(-1), torch.int64, "t")
    dev = x.device
    N = int(x.shape[0])
    fx, fy = int(input_width / output_width), int(input_height / output_height)
    cells = output_height * output_width
    if change_map is None:
        change_map = torch.zeros((output_height, output_width), dtype=torch.float32, device=dev)
    _lib.require_cuda(change_map, "change_map")
    assert change_map.dtype == torch.float32 and change_map.is_contiguous() and change_map.numel() == cells
    nb = int(lib.dagr_scan_blocks(max(N, cells) + 1)) + 2
    cell, tmp, srt = _i32(N, dev), _i32(N, dev), _i32(N, dev)
    count = torch.zeros(cells + 1, dtype=torch.int32, device=dev)
    start, blocksums = _i32(cells + 2, dev), _i32(nb, dev)
    mask = torch.zeros(max(N, 1), dtype=torch.uint8, device=dev)
    st = _lib.stream_ptr()
    _lib.check(lib.dagr_downsample_events(_lib.ptr(x), _lib.ptr(y), _lib.ptr(p), N, fx, fy, output_width, output_height,
                                          _lib.ptr(change_map), _lib.ptr(cell), _lib.ptr(tmp), _lib.ptr(srt), _lib.ptr(count),
                                          _lib.ptr(start), _lib.ptr(blocksums), _lib.ptr(mask), st), "downsample_events")
    flag, pos = _i32(N, dev), _i32(N + 1, dev)
    xo = torch.empty(max(N, 1), dtype=torch.int16, device=dev)
    yo = torch.empty(max(N, 1), dtype=torch.int16, device=dev)
    to = torch.empty(max(N, 1), dtype=torch.int64, device=dev)
    po = torch.empty(max(N, 1), dtype=torch.int8, device=dev)
    n_out = torch.zeros(1, dtype=torch.int32, device=dev)
    _lib.check(lib.dagr_compact_events(_lib.ptr(mask), N, _lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), fx, fy,
                                       _lib.ptr(flag), _lib.ptr(pos), _lib.ptr(blocksums), _lib.ptr(xo), _lib.ptr(yo),
                                       _lib.ptr(to), _lib.ptr(po), _lib.ptr(n_out), st), "compact_events")
    M = int(n_out.item())                                       # the one host sync: output length
    return dict(x=xo[:M], y=yo[:M], t=to[:M], p=po[:M]), change_map


def ingest_window(events: Dict[str, torch.Tensor], width: int, height: int, time_window: int = 1_000_000,
                  t_cut: Optional[int] = None, sample: int = 0, p_is_01: bool = True):
    """raw events of one sample (x, y u16; t int64 us; p in {0,1} as stored in the DSEC files, or +-1 with
    p_is_01=False) -> (batch int32[M], pos_denorm int32[M,3], polarity float32[M])."""
    lib = _lib.load()
    x, y = _xy16(events["x"], "x"), _xy16(events["y"], "y")
    p = _as(events["p"].reshape(-1), torch.int8, "p")
    t = _as(events["t"].reshape(-1), torch.int64, "t")
    dev = x.device
    N = int(x.shape[0])
    nb = int(lib.dagr_scan_blocks(N + 1)) + 2
    flag, pos, blocksums = _i32(N, dev), _i32(N + 1, dev), _i32(nb, dev)
    tlast = torch.zeros(1, dtype=torch.int64, device=dev)
    batch_o = _i32(N, dev)
    pos_o = torch.empty((max(N, 1), 3), dtype=torch.int32, device=dev)
    feat_o = torch.empty(max(N, 1), dtype=torch.float32, device=dev)
    n_out = torch.zeros(1, dtype=torch.int32, device=dev)
    cut = (1 << 62) if t_cut is None else int(t_cut)
    _lib.check(lib.dagr_ingest_events(_lib.ptr(x), _lib.ptr(y), _lib.ptr(t), _lib.ptr(p), N, 1 if p_is_01 else 0, int(width),
                                      int(height), int(time_window), cut, int(sample), _lib.ptr(flag), _lib.ptr(pos),
                                      _lib.ptr(blocksums), _lib.ptr(tlast), _lib.ptr(batch_o), _lib.ptr(pos_o), _lib.ptr(feat_o),
                                      _lib.ptr(n_out), _lib.stream_ptr()), "ingest_events")
    M = int(n_out.item())
    return batch_o[:M], pos_o[:M], feat_o[:M]


def frame_lut(device) -> torch.Tensor:
    """f32[256] u8 -> f32 table of the float frame form: torch's own `.float() / 255.0` on the device, so a table lookup
    has the bits of the division format_data applies."""
    return torch.arange(256, dtype=torch.uint8, device=device).float() / 255.0


def preprocess_frames(frames: torch.Tensor, height: int, width: int, scale: int, lut: Optional[torch.Tensor] = None):
    """dagr_frame_preprocess on the current stream: u8 [F, sh, sw, 3] contiguous CUDA -> u8 [F, 3, height, width], or f32
    through `lut` (frame_lut) when it is given.  Raises RuntimeError on a shape the kernel refuses."""
    lib = _lib.load()
    _lib.require_cuda(frames, "frames")
    if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
        raise ValueError(f"frames {tuple(frames.shape)} {frames.dtype}: expected u8 [F, sh, sw, 3]")
    F, sh, sw = (int(v) for v in frames.shape[:3])
    out = torch.empty((F, 3, height, width), dtype=torch.uint8 if lut is None else torch.float32, device=frames.device)
    _lib.check(lib.dagr_frame_preprocess(_lib.ptr(frames), F, sh, sw, int(scale), int(height), int(width),
                                         _lib.ptr(out) if lut is None else None, None if lut is None else _lib.ptr(out),
                                         _lib.ptr(lut), _lib.stream_ptr()), "frame_preprocess")
    return out


def preprocess_image(frames_u8: torch.Tensor, height: int, width: int, scale: int) -> torch.Tensor:
    """the reference's DSEC.preprocess_image (dsec_data.py:149-154) on the device: camera frames u8 [F, sh, sw, 3] or
    [sh, sw, 3] (HWC, CUDA, the camera's channel order, passed through) -> u8 [F, 3, height, width], the `data.image` the
    model was trained on.  Rows from scale * height on are cropped, then the frame is resized by the integer factor
    `scale` with OpenCV's INTER_CUBIC arithmetic (sw == scale * width, sh >= scale * height; other ratios raise).  No host
    sync."""
    f = frames_u8.unsqueeze(0) if frames_u8.dim() == 3 else frames_u8
    return preprocess_frames(f.contiguous(), height, width, scale)


def collate(samples, width: int, height: int, time_window: int = 1_000_000) -> EventBatch:
    """list of ingest_window results (sample index = list position) -> a Batch for `DAGR.forward`: `pos_denorm` carries
    the integer coordinates (ev_tgn.py:12-13), `pos` their fp32 normalisation for callers that read it."""
    batch = torch.cat([s[0] for s in samples])
    den = torch.cat([s[1] for s in samples])
    feat = torch.cat([s[2] for s in samples])
    dev = den.device
    B = len(samples)
    norm = torch.tensor([width, height, time_window], dtype=torch.float32, device=dev)
    return EventBatch(x=feat.view(-1, 1), pos=den.float() / norm, pos_denorm=den, batch=batch.long(),
                      width=torch.full((B,), width, device=dev), height=torch.full((B,), height, device=dev),
                      time_window=torch.full((B,), time_window, device=dev), num_graphs=B,
                      dims=(int(width), int(height), int(time_window)))
