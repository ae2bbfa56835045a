"""DAGR top module (reference: src/dagr/model/networks/dagr.py:14-312) -- same constructor, forward(),
cache_luts() and state_dict layout; the arithmetic runs in hand-written sm_90a kernels through
dagr_b200.engine.Engine.  There is no CPU path: forward() on CPU tensors raises.
"""
from __future__ import annotations

import argparse
from typing import List

import numpy as np
import torch
from torch import nn

from .layers import ConvBlock, SplineConvToDense
from .net import Net
from .yolox_compat import YOLOX, YOLOXHead


def voxel_size_to_params(pooling_layer, height, width):
    """src/dagr/model/utils.py:112-116."""
    rx = int(np.ceil(2 * pooling_layer.voxel_size[0].cpu().numpy() * width))
    ry = int(np.ceil(2 * pooling_layer.voxel_size[1].cpu().numpy() * height))
    M = pooling_layer.transform.max
    return rx, ry, M


class CNNHead(YOLOXHead):
    """dagr.py:106-122 (dense cuDNN path)."""

    def forward(self, xin):
        outputs = dict(cls_output=[], reg_output=[], obj_output=[])
        for k, (cls_conv, reg_conv, x) in enumerate(zip(self.cls_convs, self.reg_convs, xin)):
            x = self.stems[k](x)
            cls_feat = cls_conv(x)
            reg_feat = reg_conv(x)
            outputs["cls_output"].append(self.cls_preds[k](cls_feat))
            outputs["reg_output"].append(self.reg_preds[k](reg_feat))
            outputs["obj_output"].append(self.obj_preds[k](reg_feat))
        return outputs


class GNNHead(YOLOXHead):
    def __init__(self, num_classes, strides=(8, 16, 32), in_channels=(256, 512, 1024), in_channels_cnn=(256, 512, 1024),
                 act="silu", depthwise=False, pretrain_cnn=False, args=None):
        YOLOXHead.__init__(self, num_classes, args.yolo_stem_width, strides, in_channels, act, depthwise)
        self.pretrain_cnn = pretrain_cnn
        self.num_scales = args.num_scales
        self.use_image = bool(getattr(args, "use_image", False))
        self.batch_size = args.batch_size
        self.no_events = bool(getattr(args, "no_events", False))
        self.in_channels = list(in_channels)
        self.n_anchors = 1
        self.num_classes = num_classes
        n_reg = max(in_channels)
        self.stem1 = ConvBlock(in_channels=in_channels[0], out_channels=n_reg, args=args)
        self.cls_conv1 = ConvBlock(in_channels=n_reg, out_channels=n_reg, args=args)
        self.cls_pred1 = SplineConvToDense(n_reg, self.n_anchors * self.num_classes, bias=True, args=args)
        self.reg_conv1 = ConvBlock(in_channels=n_reg, out_channels=n_reg, args=args)
        self.reg_pred1 = SplineConvToDense(n_reg, 4, bias=True, args=args)
        self.obj_pred1 = SplineConvToDense(n_reg, self.n_anchors, bias=True, args=args)
        if self.num_scales > 1:
            self.stem2 = ConvBlock(in_channels=in_channels[1], out_channels=n_reg, args=args)
            self.cls_conv2 = ConvBlock(in_channels=n_reg, out_channels=n_reg, args=args)
            self.cls_pred2 = SplineConvToDense(n_reg, self.n_anchors * self.num_classes, bias=True, args=args)
            self.reg_conv2 = ConvBlock(in_channels=n_reg, out_channels=n_reg, args=args)
            self.reg_pred2 = SplineConvToDense(n_reg, 4, bias=True, args=args)
            self.obj_pred2 = SplineConvToDense(n_reg, self.n_anchors, bias=True, args=args)
        if self.use_image:
            self.cnn_head = CNNHead(num_classes=num_classes, strides=strides, in_channels=in_channels_cnn)
        self.strides = strides


class DAGR(YOLOX):
    def __init__(self, args, height, width):
        self.conf_threshold = 0.001
        self.nms_threshold = 0.65
        self.height = height
        self.width = width
        _defaults = dict(use_image=False, no_events=False, pretrain_cnn=False, keep_temporal_ordering=False,
                         activation="relu", edge_attr_dim=2, aggr="sum", kernel_size=5, pooling_aggr="max",
                         base_width=0.5, after_pool_width=1, dataset="dsec", num_scales=2,
                         pooling_dim_at_output="5x7", max_neighbors=16, radius=0.01, img_net="resnet18")
        for k, v in _defaults.items():
            if k not in args:
                setattr(args, k, v)
        backbone = Net(args, height=height, width=width)
        head = GNNHead(num_classes=backbone.num_classes, in_channels=backbone.out_channels,
                       in_channels_cnn=backbone.out_channels_cnn, strides=backbone.strides,
                       pretrain_cnn=args.pretrain_cnn, args=args)
        super().__init__(backbone=backbone, head=head)
        self.args = args
        self.time_window = int(getattr(args, "time_window_us", 1000000))
        self._engine = None
        self._async = None
        self._image_branch = None
        self.image_graph = True         # dense image branch as a replayed CUDA graph on a side stream (model/image_branch.py)
        self.keep_stream = False        # True: forward(reset=True) starts a stream that forward(reset=False) extends
        self.image_precision = "tf32"   # image branch precision, see the property
        if "img_net_checkpoint" in args:
            sd = torch.load(args.img_net_checkpoint, map_location="cpu")["ema"]
            for name in ("backbone.net.", "head.cnn_head."):
                sub = self
                for a in name.split(".")[:-1]:
                    sub = getattr(sub, a)
                sub.load_state_dict({k.replace(name, ""): v for k, v in sd.items() if name in k})

    # engines hold ctypes handles / CUDA workspaces: never deep-copied or pickled with the module
    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k in ("_engine", "_async", "_image_branch") else copy.deepcopy(v, memo)
        return new

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_engine"] = None
        d["_async"] = None
        d["_image_branch"] = None
        return d

    # packed weights follow the module's tensors: repack after anything that can replace or rewrite them
    def _apply(self, fn, *a, **kw):
        out = super()._apply(fn, *a, **kw)
        if getattr(self, "_engine", None) is not None:
            self._engine.invalidate()
        if getattr(self, "_image_branch", None) is not None:
            self._image_branch.invalidate()                 # captured graphs hold the old parameter storages
        return out

    def load_state_dict(self, *a, **kw):
        out = super().load_state_dict(*a, **kw)
        if getattr(self, "_engine", None) is not None:
            self._engine.invalidate()
        if getattr(self, "_image_branch", None) is not None:
            self._image_branch.invalidate()
        return out

    @property
    def image_precision(self) -> str:
        """precision of the dense image branch (--use_image): "tf32" (default) runs the model's own fp32 trunk and CNN head
        with TF32 convolutions and fp32 NCHW feature maps; "bf16" runs a bf16, channels_last copy of them under autocast,
        whose feature taps stay bf16 NHWC and are sampled by the bf16 forms of the event-level image kernels (everything
        downstream of the samples stays fp32).  Any other value raises ValueError.  model(data) reads it per call; AsyncDAGR
        and the fusion streaming detectors read it once, when they are constructed."""
        return self.__dict__.get("_image_precision", "tf32")

    @image_precision.setter
    def image_precision(self, value):
        from .image_branch import PRECISIONS
        if value not in PRECISIONS:
            raise ValueError(f"image_precision {value!r}: expected one of {PRECISIONS}")
        self.__dict__["_image_precision"] = value

    @property
    def engine(self):
        if self._engine is None:
            from ..engine import Engine
            self._engine = Engine(self)
        return self._engine

    def cache_luts(self, width, height, radius):
        """dagr.py:37-72 (records LUT parameters; see MySplineConv.init_lut)."""
        bb, hd = self.backbone, self.head
        if self._engine is not None:
            self._engine.invalidate()
        M = 2 * float(int(radius * width + 2) / width)
        r = int(radius * width + 1)
        bb.conv_block1.conv_block1.conv.init_lut(height=height, width=width, Mx=M, rx=r)
        bb.conv_block1.conv_block2.conv.init_lut(height=height, width=width, Mx=M, rx=r)
        for pool, layer in ((bb.pool1, bb.layer2), (bb.pool2, bb.layer3), (bb.pool3, bb.layer4), (bb.pool4, bb.layer5)):
            rx, ry, M = voxel_size_to_params(pool, height, width)
            layer.conv_block1.conv.init_lut(height=height, width=width, Mx=M, rx=rx, ry=ry)
            layer.conv_block2.conv.init_lut(height=height, width=width, Mx=M, rx=rx, ry=ry)
            if pool is bb.pool3 or (pool is bb.pool4 and hd.num_scales > 1):
                sfx = "1" if pool is bb.pool3 else "2"
                for n in ("stem", "cls_conv", "reg_conv"):
                    getattr(hd, n + sfx).conv.init_lut(height=height, width=width, Mx=M, rx=rx, ry=ry)
                for n in ("cls_pred", "reg_pred", "obj_pred"):
                    getattr(hd, n + sfx).init_lut(height=height, width=width, Mx=M, rx=rx, ry=ry)

    # ------------------------------------------------------------------------------------------
    def _prepare_events(self, x):
        """Batch -> (batch int32[N], pos int32[N,3], polarity fp32[N]) on the device."""
        from .. import _lib
        dev = x.pos.device
        if dev.type != "cuda":
            raise RuntimeError("dagr_b200: DAGR.forward needs CUDA tensors (there is no CPU fallback)")
        dims = getattr(x, "dims", None)                     # host-side (W, H, T) when the batch carries it: no sync
        if dims is not None:
            W, H, T = (int(v) for v in dims)
        else:
            W, H = int(x.width[0]), int(x.height[0])
            T = int(x.time_window[0]) if hasattr(x, "time_window") else self.time_window
        if getattr(x, "batch", None) is None:
            x.batch = torch.zeros(len(x.pos), dtype=torch.long, device=dev)
        N = int(x.pos.shape[0])
        lib = self.engine.lib
        xf = x.x
        fused = (not (hasattr(x, "pos_denorm") and x.pos_denorm is not None) and N > 0 and x.pos.dtype == torch.float32
                 and x.pos.is_contiguous() and x.batch.dtype == torch.int64 and x.batch.is_contiguous() and xf.dtype == torch.float32
                 and xf.dim() in (1, 2) and xf.stride(-1) == 1 and (xf.dim() == 1 or xf.stride(0) == xf.shape[1]))
        if fused:
            # one launch: denormalize_pos + batch.int() + polarity column (no at:: cast / copy kernels on the call path)
            pos_i = torch.empty((N, 3), dtype=torch.int32, device=dev)
            batch_i = torch.empty(N, dtype=torch.int32, device=dev)
            feat = torch.empty(N, dtype=torch.float32, device=dev)
            ldx = 1 if xf.dim() == 1 else int(xf.shape[1])
            _lib.check(lib.dagr_prepare_events(_lib.ptr(x.pos), _lib.ptr(x.batch), _lib.ptr(xf), ldx, N, W, H, T, _lib.ptr(pos_i),
                                               _lib.ptr(batch_i), _lib.ptr(feat), _lib.stream_ptr()), "prepare_events")
            self.engine.launches += 1
            return batch_i, pos_i, feat, W, H
        if hasattr(x, "pos_denorm") and x.pos_denorm is not None:               # ev_tgn.py:12-13
            pos_i = x.pos_denorm.int().contiguous()
        else:
            pos_f = x.pos.float().contiguous()
            pos_i = torch.empty((N, 3), dtype=torch.int32, device=dev)
            _lib.check(lib.dagr_denormalize_pos(_lib.ptr(pos_f), N, W, H, T, _lib.ptr(pos_i), _lib.stream_ptr()),
                       "denormalize_pos")
        batch_i = x.batch.int().contiguous()
        feat = x.x.float().reshape(N, -1)[:, 0].contiguous() if N > 0 else torch.zeros(0, device=dev)
        return batch_i, pos_i, feat, W, H

    def forward_decoded(self, x, reset=True):
        """backbone + head up to decode_outputs: [B, n_anchors, 5 + num_classes]."""
        if not reset:
            # incremental call sequence of the reference (evaluate_flops.py:115-116: forward(reset=True) then
            # forward(new events, reset=False)): append to the stream started by the last reset=True forward
            if self._async is None:
                raise RuntimeError("forward(reset=False) must follow a forward(reset=True, ...) made with keep_stream=True "
                                   "or use dagr_b200.asynchronous.AsyncDAGR directly")
            return self._async.step_decoded(x, batch_size=int(getattr(x, "num_graphs", 1) or 1))
        if self.keep_stream:
            from ..asynchronous import AsyncDAGR
            self._async = AsyncDAGR(self)
            return self._async.step_decoded(x, batch_size=int(getattr(x, "num_graphs", 1) or 1))
        batch_i, pos_i, feat, W, H = self._prepare_events(x)
        B = int(getattr(x, "num_graphs", 0) or (int(x.batch.max()) + 1 if len(x.batch) else 1))
        image_feats = image_outs = image_event = None
        if self.backbone.use_image:
            # dense image trunk + CNN head stay torch/cuDNN (tensor cores allowed here only), net.py:110, dagr.py:205-206;
            # they run on a side stream, concurrently with the sort + radius-graph kernels below
            if self._image_branch is None:
                from .image_branch import ImageBranch
                self._image_branch = ImageBranch(self)
            image_feats, image_outs, image_event = self._image_branch.run(x.image, use_graph=self.image_graph,
                                                                          precision=self.image_precision)
            self.last_image_outs, self.last_image_feats = image_outs, image_feats
            if self.head.no_events:
                # --no_events (dagr.py:284): detections from the image branch alone -- collect_outputs + decode_outputs on
                # the CNN head maps (tiny dense tensors; plain torch on the current stream)
                torch.cuda.current_stream().wait_event(image_event[1])
                return self._decode_image_only(image_outs)
        elif self.head.no_events:
            raise RuntimeError("--no_events needs --use_image (the reference would fail on the missing image branch too)")
        return self.engine.forward_events(batch_i, pos_i, feat, B, W, H, image_feats=image_feats, image_outs=image_outs,
                                          image_event=image_event)

    def _decode_image_only(self, image_outs):
        """GNNHead.collect_outputs + decode_outputs (dagr.py:292-312) for image_out['outputs']."""
        outs, grids, strides = [], [], []
        for k in range(self.head.num_scales):
            reg, obj, cls = (image_outs[n + "_output"][k] for n in ("reg", "obj", "cls"))
            o = torch.cat([reg, obj.sigmoid(), cls.sigmoid()], 1)
            h, w = o.shape[-2:]
            yv, xv = torch.meshgrid(torch.arange(h, device=o.device), torch.arange(w, device=o.device), indexing="ij")
            grids.append(torch.stack((xv, yv), 2).view(1, -1, 2).float())
            strides.append(torch.full((1, h * w, 1), float(self.backbone.strides[k]), device=o.device))
            outs.append(o.flatten(start_dim=2))
        out = torch.cat(outs, dim=2).permute(0, 2, 1).contiguous()
        grid, stride = torch.cat(grids, 1), torch.cat(strides, 1)
        out[..., :2] = (out[..., :2] + grid) * stride
        out[..., 2:4] = torch.exp(out[..., 2:4]) * stride
        return out

    def forward(self, x, reset=True, return_targets=True, filtering=True):
        if self.training:
            raise NotImplementedError("training (YOLOX losses) is out of scope of this build; call .eval()")
        x.reset = reset
        outputs = self.forward_decoded(x, reset=reset)
        det, ndet = self.engine.postprocess(outputs, self.conf_threshold, self.nms_threshold, self.width, self.height,
                                            filtering=filtering)
        self.engine.join()                                           # overlap mode: results come from the side stream
        counts = ndet.tolist()                                       # the one device->host sync of the forward
        detections = []
        for b, n in enumerate(counts):
            d = det[b, :n]
            detections.append(dict(boxes=d[:, :4], scores=d[:, 4], labels=d[:, 5].long()))
        ret = [detections]
        if return_targets and hasattr(x, "bbox") and x.bbox is not None:
            ret.append(convert_to_evaluation_format(x))
        return ret


def convert_to_evaluation_format(data):
    """src/dagr/model/utils.py:35-44 for a collated batch (bbox xywh+cls, bbox_batch)."""
    targets = []
    B = int(data.num_graphs)
    bb = data.bbox_batch if hasattr(data, "bbox_batch") else torch.zeros(len(data.bbox), dtype=torch.long)
    for b in range(B):
        bbox = data.bbox[bb == b].clone()
        bbox[:, 2:4] += bbox[:, :2]
        targets.append(dict(boxes=bbox[:, :4], labels=bbox[:, 4].long()))
    return targets
