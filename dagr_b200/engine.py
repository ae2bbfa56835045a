"""Host-side driver of the hot path: reads the nn.Module tree's tensors, owns geometry tables and
workspaces, and enqueues the sm_90a kernels of libdagr_b200.so on the current CUDA stream.

Call sequence mirrors Net.forward / GNNHead.forward (src/dagr/model/networks/net.py:108-190,
dagr.py:192-312) but the event level is fused (graph sort -> probe -> conv_a -> conv_b+pool1) and the
coarse levels run on dense voxel grids.  No host synchronisation happens inside `forward_events`.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from . import _lib
from .geometry import Geometry


def _fold_bn(bn):
    m = bn.module
    scale = (m.weight / torch.sqrt(m.running_var + m.eps)).float()
    shift = (m.bias - m.running_mean * scale).float()
    return scale.contiguous(), shift.contiguous()


def _tc_weights(lib, params, cin: int, device) -> torch.Tensor:
    """params.w / params.root (input channels 0..15) in the mma fragment order of the tensor-core conv kernels (dagr_l1_tc_weights)."""
    out = (C.c_float * _lib.L1_TC_WFRAG_FLOATS)()
    _lib.check(lib.dagr_l1_tc_weights(params.w, params.root, cin, out), "dagr_l1_tc_weights")
    return torch.frombuffer(out, dtype=torch.float32).clone().to(device)


def _l1a_tc_weights(lib, params, device) -> torch.Tensor:
    """params.w / params.root of conv_block1.conv_block1's event channels in the mma fragment order of the tensor-core build
    kernel (dagr_l1a_tc_weights)."""
    out = (C.c_float * _lib.L1A_TC_WFRAG_FLOATS)()
    _lib.check(lib.dagr_l1a_tc_weights(params, out), "dagr_l1a_tc_weights")
    return torch.frombuffer(out, dtype=torch.float32).clone().to(device)


def _fill(arr, t: torch.Tensor):
    flat = t.detach().float().cpu().contiguous().view(-1)
    assert flat.numel() == len(arr), (flat.numel(), len(arr))
    C.memmove(arr, flat.data_ptr(), flat.numel() * 4)


def _image_format(image_feats) -> torch.dtype:
    """the format of the image taps, which selects the sampling entry points: fp32 NCHW (the TF32 image branch) or bf16 in
    channels_last memory format (NHWC, the bf16 branch, DAGR.image_precision); the taps of one call share it."""
    dt = image_feats[0].dtype
    if dt not in (torch.float32, torch.bfloat16) or any(f.dtype != dt for f in image_feats):
        raise ValueError(f"image_feats of dtypes {[f.dtype for f in image_feats]}: expected all float32 or all bfloat16")
    if dt == torch.bfloat16 and not all(f.dim() == 4 and f.is_contiguous(memory_format=torch.channels_last) for f in image_feats):
        raise ValueError("bfloat16 image_feats must be [B, C, h, w] tensors in channels_last memory format (NHWC)")
    return dt


@dataclass(frozen=True, eq=False)
class _Taps:
    """the image taps of one forward_events call and the entry points that sample them.  Each image kernel's entry point is
    chosen here: first the format (fp32 NCHW, or bf16 channels_last: the _bf16 forms), then the mode: a plane per sample
    (the _planes forms), x0 bounded by the live total (_live), the running voxel max of an incremental call (_inc), or
    plain.  Call sites pass the arguments every form takes."""
    feats: list                        # the five taps [B or P, C, h, w]: conv1 (x0), layer1 (voxel max), layer2..4 (coarse)
    outs: Optional[dict]               # CNN head maps: "{cls,reg,obj}_output" -> one fp32 [B or P, C, ny, nx] per scale
    fmt: torch.dtype                   # _image_format(feats)
    planes: Optional[tuple] = None     # (plane table int32 on the device, stride): sample b reads plane table[b * stride]
    live: bool = False                 # ring sorts: N is the capacity, x0 is bounded by the live total start[NK]
    state: object = None               # the StreamState of an incremental call (voxel max into state.imgmax)
    min_idx: int = 0

    @property
    def sfx(self):
        return "_bf16" if self.fmt == torch.bfloat16 else ""

    def _plane_args(self, t):
        return (int(t.shape[0]), self.planes[0], int(self.planes[1])) if self.planes is not None else ()

    def x0(self, eng, g, N, start, xyb, feat_s, x0, st):
        """the conv1 tap at every node; incremental steps resample every node too: a new node's conv reads the x0 rows of
        its older neighbours."""
        f = self.feats[0]
        img = (f,) + ((int(f.shape[1]),) if self.sfx else ()) + (int(f.shape[2]), int(f.shape[3]))  # bf16 takes C
        if self.planes is not None:
            form, args = "_planes", (start, xyb, feat_s, *img, *self._plane_args(f))
        elif self.live:
            # N = ring capacity: positions behind the live total hold stale xyb words, so the launch is bounded by the
            # total the sort wrote (start[NK]); the synchronous path keeps the unbounded form (N is the live count there)
            form, args = "_live", (start, xyb, feat_s, *img)
        else:
            form, args = "", (xyb, feat_s, *img)
        eng._run("l1_x0_image", getattr(eng.lib, "dagr_l1_x0_image" + form + self.sfx), g, N, *args, x0, st)

    def voxel_max(self, eng, g, N, start, xyb, ti, xg, ldx, c0, pool_mean, st):
        """the per-voxel max of the layer1 tap's samples into xg[:, c0:] (sampling_skip before pool1, net.py:128-131)."""
        f = self.feats[1]
        img = (f, int(f.shape[1]), int(f.shape[2]), int(f.shape[3]))
        if self.state is not None:            # running per-voxel max of the samples, new events only
            label, form, args = "voxel_sample_max_inc", "_inc", (ti, *img, self.min_idx, self.state.imgmax)
        else:
            label, form, args = "voxel_sample_max", "_planes" if self.planes is not None else "", (*img, *self._plane_args(f))
        eng._run(label, getattr(eng.lib, "dagr_voxel_sample_max" + form + self.sfx), g, N, start, xyb, *args, xg, ldx, c0,
                 pool_mean, st)

    def sample_features(self, eng, k, posx, posy, bidx, n, width, height, out, ldo, c0, st):
        """tap k sampled at n grid nodes into out[:, c0:]."""
        f = self.feats[k]
        form = "_planes" if self.planes is not None else ""
        eng._run("sample_features", getattr(eng.lib, "dagr_sample_features" + form + self.sfx), f,
                 *(self._plane_args(f) or (int(f.shape[0]),)), int(f.shape[1]), int(f.shape[2]), int(f.shape[3]), posx, posy,
                 bidx, n, width, height, out, ldo, c0, st)

    def head_maps(self, k):
        """-> (form, maps, plane arguments) of dagr_head_finish[form] at scale k: the CNN head maps added to the graph
        head's cls / reg / obj outputs (fp32 in every format; None without maps)."""
        adds = {n: None if self.outs is None else self.outs[n + "_output"][k].float().contiguous() for n in ("cls", "reg", "obj")}
        return ("_planes" if self.planes is not None else ""), adds, self._plane_args(adds["cls"])


def _overlaps(overlap: bool, profiling: bool, use_graphs: bool) -> bool:
    """whether a plain forward runs its coarse stack + NMS on the side stream (Engine.overlap): only with graphs on and
    per-op timing off."""
    return bool(overlap and not profiling and use_graphs)


@dataclass(frozen=True, eq=False)
class _Mode:
    """how one forward_events call runs (resolve_mode)."""
    sort: str                          # "batch" (dagr_graph_sort), "ring" (one ring) or "rings" (S rings of N / S slots)
    ring: Optional[torch.Tensor]       # the ring control block: int32[8], or int32[S+1][8] for S rings
    streams: int                       # S of "rings", else 1
    state: object                      # the StreamState of an incremental call, else None
    min_idx: int                       # incremental: the arrival indices below it were processed by earlier steps
    taps: Optional[_Taps]              # image fusion
    overlap: bool                      # coarse stack + NMS on the side stream, double-buffered hand-off
    capture: bool                      # coarse stack replayed as one captured CUDA graph
    fixed: bool                        # rings or incremental: "auto" queues no voxels for the dense kernels (_dense_policy)


def resolve_mode(B: int, N: int, image_feats=None, image_outs=None, stream_state=None, n_old: int = 0, ring=None,
                 ring_streams=None, image_planes=None, *, overlap=False, profiling=False, use_graphs=True,
                 keep_node_features=False) -> _Mode:
    """the mode of one Engine.forward_events call, from its arguments and the engine's switches.  Host only, no CUDA: every
    refusal comes before any device work."""
    if ring_streams is not None and (ring is None or int(ring_streams) != int(B) or N % int(ring_streams)):
        raise ValueError(f"ring_streams={ring_streams} needs a ring control block, B == ring_streams and N a multiple of it "
                         f"(B={B}, N={N})")
    if stream_state is not None and ring is not None:
        raise ValueError("stream_state with a ring: an incremental call appends to one event history, whose arrival indices "
                         "a ring shifts with every eviction")
    if image_planes is not None:
        if image_feats is None or image_outs is None:
            raise ValueError("image_planes selects a frame per sample: it needs image_feats and image_outs")
        if keep_node_features:
            raise ValueError("keep_node_features: the dense head maps (dagr_grid_to_dense) have no plane mode")
        if stream_state is not None:
            raise ValueError("stream_state with image_planes: the running voxel max (dagr_voxel_sample_max_inc) has no plane "
                             "mode")
    min_idx = int(n_old) if stream_state is not None else 0
    taps = None
    if image_feats is not None:
        # the taps' format picks the fp32 or the bf16 sampling entry points
        taps = _Taps(image_feats, image_outs, _image_format(image_feats),
                     None if image_planes is None else (image_planes[0], int(image_planes[1])), ring is not None,
                     stream_state, min_idx)
    ov = _overlaps(overlap, profiling, use_graphs) and ring is None and stream_state is None and image_planes is None
    return _Mode(sort="batch" if ring is None else "ring" if ring_streams is None else "rings", ring=ring,
                 streams=1 if ring_streams is None else int(ring_streams), state=stream_state, min_idx=min_idx, taps=taps,
                 overlap=ov,
                 # with image fusion only the overlapped step is captured (the serial hybrid forward stays eager)
                 capture=bool(use_graphs and not profiling and ring is None and (ov or taps is None)),
                 fixed=ring is not None or stream_state is not None)


class _ConvPack:
    def __init__(self, conv, norm=None, relu=False, dev=None):
        self.cin, self.cout = conv.in_channels, conv.out_channels
        self.weight = conv.weight.detach().float().contiguous().to(dev)
        self.rootT = conv.lin.weight.detach().float().t().contiguous().to(dev)
        self.bias = conv.bias.detach().float().contiguous().to(dev) if conv.bias is not None else None
        if norm is not None:
            s, b = _fold_bn(norm)
            self.scale, self.shift = s.detach().to(dev), b.detach().to(dev)
        else:
            self.scale = self.shift = None
        self.relu = relu


def _merge_packs(a: "_ConvPack", b: "_ConvPack") -> "_ConvPack":
    """two SplineConvs over the SAME input evaluated as one conv with the output channels side by side."""
    m = _ConvPack.__new__(_ConvPack)
    assert a.cin == b.cin and a.relu == b.relu and (a.bias is None) == (b.bias is None) and (a.scale is None) == (b.scale is None)
    m.cin, m.cout = a.cin, a.cout + b.cout
    m.weight = torch.cat([a.weight, b.weight], dim=2).contiguous()
    m.rootT = torch.cat([a.rootT, b.rootT], dim=1).contiguous()
    m.bias = None if a.bias is None else torch.cat([a.bias, b.bias]).contiguous()
    m.scale = None if a.scale is None else torch.cat([a.scale, b.scale]).contiguous()
    m.shift = None if a.shift is None else torch.cat([a.shift, b.shift]).contiguous()
    m.relu = a.relu
    return m


class _LayerPack:
    def __init__(self, layer, relu, dev):
        self.a = _ConvPack(layer.conv_block1.conv, layer.conv_block1.norm, relu, dev)
        self.b = _ConvPack(layer.conv_block2.conv, layer.conv_block2.norm, relu, dev)
        self.skipT = layer.conv_block2.lin.mlp.weight.detach().float().t().contiguous().to(dev)
        s, b = _fold_bn(layer.conv_block2.norm_skip)
        self.sscale, self.sshift = s.detach().to(dev), b.detach().to(dev)


class GridState:
    """one voxel-grid level: valid count, rounded pixel position, t statistics, in-edge mask, features."""

    def __init__(self, level, cells, dev):
        self.level = level
        self.cells = cells
        self.cnt = torch.empty(cells, dtype=torch.int32, device=dev)
        self.pxy = torch.empty((cells, 2), dtype=torch.int32, device=dev)
        self.tmean = torch.empty(cells, dtype=torch.float32, device=dev)
        self.tmax = torch.empty(cells, dtype=torch.float32, device=dev)
        self.mask = None
        self.x = None


class _WsView:
    """workspace seen by one forward: the event-level buffers are shared, everything the coarse stack touches
    (zero-on-entry accumulators, grid states, pooled buffers, the captured CUDA graph) belongs to a SLOT so that
    the coarse stack of step i can run on a side stream while the event-level kernels of step i+1 execute."""
    _SLOT_KEYS = ("zero_buf", "grids", "pool", "graph", "graph_warm", "graph_key")

    def __init__(self, base: dict, slot: dict):
        self.base, self.slot = base, slot

    def __getitem__(self, k):
        return self.slot[k] if k in self._SLOT_KEYS else self.base[k]

    def __setitem__(self, k, v):
        (self.slot if k in self._SLOT_KEYS else self.base)[k] = v

    def __contains__(self, k):
        return k in (self.slot if k in self._SLOT_KEYS else self.base)

    def get(self, k, default=None):
        return (self.slot if k in self._SLOT_KEYS else self.base).get(k, default)


class Engine:
    def __init__(self, model):
        self.model = model
        self.lib = _lib.load()
        self._geoms: Dict[tuple, Geometry] = {}
        self._pack = None
        self._pack_key = None
        self._pack_gen = 0                   # bumped by every repack: captured graphs of older packs are never replayed
        self._sentinels = None
        self._ws: Dict[tuple, dict] = {}
        self.keep_node_features = False      # debug / parity: materialise per-event activations
        self.use_graphs = True               # replay the fixed-shape coarse stack as a CUDA graph
        # voxels beyond the per-voxel kernels' staging capacity (moving edges): "auto" = the kernels always COUNT them; once a
        # forward has seen some, the following forwards queue them for the persistent dense kernels (two more launches,
        # even when empty, which is why uniform streams do not pay for them); True / False force the behaviour (tests, A/B)
        self.dense_worklists = "auto"
        self._dense = {}                     # workspace id -> dict(defer=[build, conv_a, conv_b], host=pinned i32[8], event, quiet)
        self.last = {}
        self.launches = 0                    # kernels of libdagr_b200.so enqueued so far
        self.prof = None                     # dict name -> [(start_evt, end_evt)] when per-op timing is on
        # overlap=True: the coarse stack + NMS of step i run on a side stream (double-buffered hand-off) while the
        # caller's stream already executes the event-level kernels of step i+1.  Results of a step are then valid only
        # after join() (or on result_stream()); they stay valid until the second next forward.  Plain reset=True
        # batches, events-only or with image taps (whose last reader is then the side stream: a caller that rewrites
        # them waits for _done[slot], see next_slot()); streaming, incremental and per-sample-frame forwards silently
        # take the serial path.
        self.overlap = False
        self._cstream = None
        self._fstream = None                 # forked branch of the coarse stack (first head scale)
        self._slot = 0
        self._done = [None, None]
        self._out_slot = {}

    # kernels enqueued by each C-ABI call (see csrc/*.cu)
    _NKERNELS = dict(dagr_graph_sort=6, dagr_graph_sort_ring=6, dagr_stream_push=2, dagr_graph_sort_rings=6, dagr_stream_push_multi=2, dagr_stream_ingest=1, dagr_window_gather=1, dagr_l1_build=2, dagr_l1_build_tc=2, dagr_graph_export=5, dagr_l1_conv_b_pool_voxel_tc=2, dagr_l1_x0_image=1, dagr_l1_x0_image_live=1, dagr_xa_permute=1, dagr_l1_conv_a_image_tc=2, dagr_voxel_sample_max=1,
                     dagr_l1_conv_a_image_inc=2, dagr_voxel_sample_max_inc=1,
                     dagr_l1_x0_image_planes=1, dagr_voxel_sample_max_planes=1, dagr_sample_features_planes=1, dagr_head_finish_planes=1,
                     dagr_grid_cat_pos=1, dagr_grid_conv=1, dagr_grid_linear_bn=1, dagr_grid_pool=1,
                     dagr_grid_pool_finalize=1, dagr_grid_temporal_filter=1, dagr_grid_to_dense=1, dagr_head_finish=1,
                     dagr_postprocess_nms=1, dagr_sample_features=1, dagr_denormalize_pos=1,
                     dagr_l1_x0_image_bf16=1, dagr_l1_x0_image_live_bf16=1, dagr_l1_x0_image_planes_bf16=1, dagr_voxel_sample_max_bf16=1,
                     dagr_voxel_sample_max_inc_bf16=1, dagr_voxel_sample_max_planes_bf16=1, dagr_sample_features_bf16=1,
                     dagr_sample_features_planes_bf16=1)

    def _run(self, label, fn, *args):
        if self.prof is not None:
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
        _lib.check(fn(*args), label)
        self.launches += self._NKERNELS.get(fn.__name__, 1)
        if self.prof is not None:
            e1.record()
            self.prof.setdefault(label, []).append((e0, e1))

    def prof_summary(self):
        """mean milliseconds per op label (call after torch.cuda.synchronize())."""
        out = {}
        for k, evs in (self.prof or {}).items():
            ts = [a.elapsed_time(b) for a, b in evs]
            out[k] = dict(ms=sum(ts) / len(ts), calls=len(ts))
        return out

    # ------------------------------------------------------------------------------------------
    def geometry(self, W, H, B, device) -> Geometry:
        key = (int(W), int(H), int(B), str(device))
        g = self._geoms.get(key)
        if g is None:
            a = self.model.args
            g = Geometry(W, H, B, radius=a.radius, time_window=self.model.time_window,
                         max_neighbors=a.max_neighbors, max_queue_size=self.model.backbone.events_to_graph.max_queue_size,
                         pooling_dim_at_output=a.pooling_dim_at_output, kernel_size=getattr(a, "kernel_size", 5),
                         device=device)
            self._geoms[key] = g
        return g

    def _params_key(self):
        """cheap change detector for the packed weights: (data_ptr, version) of a few sentinel tensors spread over the
        module tree (a full scan of the ~280 state tensors every forward is not free).  `invalidate()` forces a repack;
        DAGR calls it from load_state_dict / .to() / cache_luts()."""
        if self._sentinels is None:
            ts = [t for t in self.model.state_dict().values() if t.dtype.is_floating_point]
            step = max(1, len(ts) // 12)
            self._sentinels = ts[::step] + ts[-1:]
        return tuple((t.data_ptr(), t._version) for t in self._sentinels)

    def invalidate(self):
        self._pack = None
        self._pack_key = None
        self._sentinels = None
        self._pack_gen += 1
        for ws in self._ws.values():                         # captured coarse stacks hold pointers into the old pack
            for sw in ws.get("slots", {}).values():
                sw.pop("graph", None)
                sw.pop("graph_key", None)
                sw["graph_warm"] = 0

    def pack(self, geom: Geometry, device):
        key = (self._params_key(), tuple(geom.slots1), str(device))
        if self._pack is not None and self._pack_key == key:
            return self._pack
        if self._cstream is not None:
            self._cstream.synchronize()                      # a coarse stack in flight may still read the old weight tensors
        m = self.model
        bb, hd = m.backbone, m.head
        act = getattr(m.args, "activation", "relu")
        relu = True
        l1 = bb.conv_block1
        ca, cb = l1.conv_block1, l1.conv_block2
        slots = torch.tensor(geom.slots1, dtype=torch.long)
        cin0 = ca.conv.in_channels
        # every shape restriction of the kernels lives in ONE C-ABI call (include/dagr_b200.h: dagr_check_config)
        if self.lib.dagr_check_config(geom.c_geom, 0, int(cin0), int(ca.conv.out_channels), str(act).encode()) != 0:
            raise NotImplementedError("dagr_b200: " + (self.lib.dagr_last_error() or b"").decode())
        pb = _lib.L1BParams()
        _fill(pb.w, cb.conv.weight.detach().cpu()[slots])                    # [15,16,16]
        _fill(pb.root, cb.conv.lin.weight.detach().cpu().t())
        s, b = _fold_bn(cb.norm); _fill(pb.scale, s); _fill(pb.shift, b)
        s, b = _fold_bn(cb.norm_skip); _fill(pb.sscale, s); _fill(pb.sshift, b)
        pb.relu = 1
        pb.pool_mean = 0 if getattr(m.args, "pooling_aggr", "max") == "max" else 1            # net.py:79 (pool1 aggr)
        for i in range(3):
            pb.xs[i] = geom.slots_x[i]
        for j in range(5):
            pb.ys[j] = geom.slots_y[j]
        pb.den_x, pb.den_y = geom.den1_x, geom.den1_y
        pk = dict(l1b=pb, l1a=None, l1img=None)
        pk["l1b_wfrag"] = _tc_weights(self.lib, pb, 16, device)
        if cin0 == 3:
            pa = _lib.L1AParams()
            _fill(pa.w, ca.conv.weight.detach().cpu()[slots])                # [15,3,16]
            _fill(pa.root, ca.conv.lin.weight.detach().cpu().t())           # [3,16]
            s, b = _fold_bn(ca.norm); _fill(pa.scale, s); _fill(pa.shift, b)
            pa.relu = 1
            _fill(pb.skip, cb.lin.mlp.weight.detach().cpu().t())            # [3,16]
            pk["l1a"] = pa
            pk["l1a_wfrag"] = _l1a_tc_weights(self.lib, pa, device)
        else:
            # input channels of the layer: [polarity, 16 image samples, x, y] (net.py:117-124).  The image channels go to the
            # TMA-staged conv (rows 0..15 of the padded 24), the three event channels to the probe kernel (they need no gather)
            order = list(range(1, 17)) + [0, 17, 18]
            pi = _lib.L1ImgParams()
            w = torch.zeros(15, 24, 16); w[:, :19] = ca.conv.weight.detach().cpu().float()[slots][:, order]
            r = torch.zeros(24, 16); r[:19] = ca.conv.lin.weight.detach().cpu().float().t()[order]
            k = torch.zeros(24, 16); k[:19] = cb.lin.mlp.weight.detach().cpu().float().t()[order]
            _fill(pi.w, w); _fill(pi.root, r); _fill(pi.skip, k)
            pe = _lib.L1AParams()                            # event-channel part: plain sums (BN / act happen after the image part)
            _fill(pe.w, ca.conv.weight.detach().cpu().float()[slots][:, [0, 17, 18]])
            _fill(pe.root, ca.conv.lin.weight.detach().cpu().float().t()[[0, 17, 18]])
            _fill(pe.scale, torch.ones(16)); _fill(pe.shift, torch.zeros(16))
            pe.relu = 0
            pk["l1a_img"] = pe
            pk["l1a_img_wfrag"] = _l1a_tc_weights(self.lib, pe, device)
            s, b = _fold_bn(ca.norm); _fill(pi.scale, s); _fill(pi.shift, b)
            s, b = _fold_bn(cb.norm_skip); _fill(pi.sscale, s); _fill(pi.sshift, b)
            pi.relu = 1
            pk["l1img"] = pi
            pk["l1img_wfrag"] = _tc_weights(self.lib, pi, 24, device)
        pk["layers"] = [_LayerPack(getattr(bb, n), relu, device) for n in ("layer2", "layer3", "layer4", "layer5")]
        heads = []
        for k in range(hd.num_scales):
            sfx = str(k + 1)
            stem, cc, rc = getattr(hd, "stem" + sfx), getattr(hd, "cls_conv" + sfx), getattr(hd, "reg_conv" + sfx)
            hp = dict(stem=_ConvPack(stem.conv, stem.norm, relu, device),
                      cls_conv=_ConvPack(cc.conv, cc.norm, relu, device),
                      reg_conv=_ConvPack(rc.conv, rc.norm, relu, device),
                      cls_pred=_ConvPack(getattr(hd, "cls_pred" + sfx), None, False, device),
                      reg_pred=_ConvPack(getattr(hd, "reg_pred" + sfx), None, False, device),
                      obj_pred=_ConvPack(getattr(hd, "obj_pred" + sfx), None, False, device))
            # convs that read the same tensor run as one launch: cls_conv | reg_conv (both on the stem output) and
            # reg_pred | obj_pred (both on the reg_conv output), dagr.py:179-190
            hp["clsreg_conv"] = _merge_packs(hp["cls_conv"], hp["reg_conv"])
            hp["regobj_pred"] = _merge_packs(hp["reg_pred"], hp["obj_pred"])
            heads.append(hp)
        pk["heads"] = heads
        self._pack_gen += 1
        self._pack, self._pack_key = pk, key
        return pk

    # ------------------------------------------------------------------------------------------
    def workspace(self, geom: Geometry, N: int, device):
        key = (id(geom), str(device))
        ws = self._ws.get(key)
        cap = 0 if ws is None else ws["cap"]
        if ws is None or N > cap:
            if self._cstream is not None:
                # the old buffers may still be read by a coarse stack on the side stream; they were allocated on the
                # caller's stream, so the caching allocator would hand them out again without waiting for that stream
                self._cstream.synchronize()
            cap = max(int(N * 1.25), 1024)
            dev = device
            nscan = max(geom.NK + 1, cap + 1)
            ws = dict(cap=cap)
            sz = _lib.EventWs()                                   # the library states its own workspace sizes (bytes)
            _lib.check(self.lib.dagr_event_workspace_bytes(geom.c_geom, cap, sz), "event_workspace_bytes")
            for name, dt in (("key", torch.int32), ("tmp", torch.int32), ("blocksums", torch.int32), ("start", torch.int32),
                             ("perm", torch.int32), ("ti", torch.int32), ("xyb", torch.int32), ("feat_s", torch.float32),
                             ("nbr", torch.int32), ("off", torch.int16), ("xa", torch.float32)):
                ws[name] = torch.empty(int(getattr(sz, name)) // torch.empty(0, dtype=dt).element_size(), dtype=dt, device=dev)
            ws["ti"] = ws["ti"].view(-1, 2)
            ws["count"] = torch.zeros(int(sz.count) // 4, dtype=torch.int32, device=dev)      # zero on entry, zero again on exit
            ws["x1"] = None
            # zero-on-entry accumulators of all levels in ONE buffer (single memset per forward)
            C_lv = self.model.backbone.output_channels          # [16, 64, C, C, C]
            sizes = {}
            off = 0

            def take(name, nbytes):
                nonlocal off
                nbytes = (nbytes + 255) // 256 * 256
                sizes[name] = (off, nbytes)
                off += nbytes

            take("cellmask", int(sz.cellmask))
            bb = self.model.backbone
            fc = list(getattr(getattr(bb, "net", None), "feature_channels", [])) if bb.use_image else []
            for lv in (1, 2, 3):
                cells = geom.cells(lv)
                Cc = C_lv[lv] + (fc[lv + 1] if bb.use_image else 0)      # channels pooled into this level (net.py:141-171)
                psz = _lib.PoolWs()
                _lib.check(self.lib.dagr_pool_workspace_bytes(cells, int(Cc), psz), "pool_workspace_bytes")
                take(f"acc{lv}", int(psz.acc))
                take(f"possum{lv}", int(psz.possum))
                take(f"ptmax{lv}", int(psz.ptmax))
                take(f"pcnt{lv}", int(psz.pcnt))
                take(f"pmask{lv}", int(psz.pmask))
            take("wl_hdr", 32)                                   # dense-voxel work lists: (count, cursor) x {build, conv_a, conv_b}
            for wl in ("wl_build", "wl_conv_a", "wl_conv_b"):     # ... and the queued voxel ids
                take(wl, int(sz.wl_ids))
            take("err", 4)
            take("flags", 16)
            ws["zero_buf"] = torch.zeros(off, dtype=torch.uint8, device=dev)
            ws["zero_slices"] = sizes
            grids = []
            for lv in range(4):
                grids.append(GridState(lv, geom.cells(lv), dev))
            ws["grids"] = grids
            ws["pool"] = {}
            self._ws[key] = ws
        return ws

    def _slot_view(self, ws: dict, slot: int, geom: Geometry, dev) -> _WsView:
        slots = ws.setdefault("slots", {})
        sw = slots.get(slot)
        if sw is None:
            if slot == 0:
                sw = dict(zero_buf=ws["zero_buf"], grids=ws["grids"], pool=ws["pool"])
            else:
                sw = dict(zero_buf=torch.zeros_like(ws["zero_buf"]), grids=[GridState(lv, geom.cells(lv), dev) for lv in range(4)],
                          pool={})
            slots[slot] = sw
        return _WsView(ws, sw)

    def next_slot(self):
        """-> (slot, event) of the next plain forward when it overlaps (overlap on, no per-op timing, graphs on), else
        None: the hand-off slot it will use and the event of the last step that read that slot (None if none did)."""
        if not _overlaps(self.overlap, self.prof is not None, self.use_graphs):
            return None
        return self._slot, self._done[self._slot]

    def join(self):
        """make the current stream wait for every coarse stack / NMS still running on the side stream."""
        cur = torch.cuda.current_stream()
        for ev in self._done:
            if ev is not None:
                cur.wait_event(ev)

    def fence(self):
        """work enqueued on result_stream() after the last forward (a collective, a copy) becomes part of that step."""
        if self.overlap and self._cstream is not None and self._out_slot:
            ev = torch.cuda.Event()
            ev.record(self._cstream)
            self._done[next(iter(self._out_slot.values()))] = ev

    def result_stream(self):
        """context manager: the stream on which the last forward's results are produced (current stream if serial)."""
        return torch.cuda.stream(self._cstream if (self.overlap and self._cstream is not None) else torch.cuda.current_stream())

    def _dense_policy(self, ws, wl_hdr, fixed: bool):
        """which of (build, conv_a_image, conv_b) hand their over-capacity voxels to the dense kernels in this forward."""
        if self.dense_worklists is True:
            return [1, 1, 1]
        if self.dense_worklists is False or fixed:
            # streaming (captured graph, one sample, <= 100 k live events): the launch list is fixed at capture time and a
            # 50 ms window of one stream stays far below the staging capacities; over-capacity voxels still work (L2 gathers)
            return [0, 0, 0]
        st = self._dense.get(id(ws.base))
        if st is None:
            st = dict(defer=[0, 0, 0], host=torch.zeros(8, dtype=torch.int32).pin_memory(), event=None, quiet=[0, 0, 0])
            self._dense[id(ws.base)] = st
        if st["event"] is not None and st["event"].query():            # counts of an earlier forward have arrived (no waiting)
            h = st["host"]
            cells = max(1, ws["grids"][0].cells)
            for k in range(3):
                # worth two extra launches (even when the list is empty) once >= 5 % of the voxels are over capacity;
                # a uniform 300 k-event sample has ~1 % of its voxels just above the conv kernel's 1344 rows
                if int(h[2 * k]) * 20 >= cells:
                    st["defer"][k], st["quiet"][k] = 1, 0
                elif st["defer"][k]:
                    st["quiet"][k] += 1
                    if st["quiet"][k] >= 16:                            # the stream calmed down: drop the two extra launches
                        st["defer"][k] = 0
            st["event"] = None
        return list(st["defer"])

    def _dense_report(self, ws, wl_hdr):
        st = self._dense.get(id(ws.base))
        if st is None or st["event"] is not None:
            return
        st["host"].copy_(wl_hdr[:8], non_blocking=True)                 # 32 bytes, no synchronisation; read by a later forward
        ev = torch.cuda.Event()
        ev.record()
        st["event"] = ev

    def _zs(self, ws, name, dtype):
        off, nbytes = ws["zero_slices"][name]
        return ws["zero_buf"][off:off + nbytes].view(dtype)

    def _buf(self, ws, name, shape, dtype, dev):
        t = ws["pool"].get(name)
        n = 1
        for s in shape:
            n *= s
        if t is None or t.numel() < n or t.dtype != dtype:
            t = torch.empty(max(n, 1), dtype=dtype, device=dev)
            ws["pool"][name] = t
        return t[:n].view(*shape)

    # ------------------------------------------------------------------------------------------
    def _grid_conv(self, geom, lv, gs: GridState, xin, pack: _ConvPack, skip, out, st, ldin=0):
        level = geom.levels[lv]
        self._run(f"grid_conv_L{lv + 1}_{pack.cin}x{pack.cout}", self.lib.dagr_grid_conv, level.grid, gs.cnt, gs.pxy, gs.mask,
                  xin, int(ldin), pack.cin, pack.cout, pack.weight, pack.rootT, pack.bias, pack.scale, pack.shift, skip,
                  1 if pack.relu else 0, level.den_x, level.den_y, out, st)

    def _layer(self, geom, lv, gs: GridState, lp: _LayerPack, ws, name, st, dev):
        level = geom.levels[lv]
        cells = gs.cells
        cx = gs.x.shape[1]
        xin = self._buf(ws, name + "_in", (cells, cx + 2), torch.float32, dev)
        self._run("cat_pos", self.lib.dagr_grid_cat_pos, level.grid, gs.cnt, gs.pxy, gs.x, cx, xin, st)
        a = self._buf(ws, name + "_a", (cells, lp.a.cout), torch.float32, dev)
        self._grid_conv(geom, lv, gs, xin, lp.a, None, a, st)
        sk = self._buf(ws, name + "_s", (cells, lp.b.cout), torch.float32, dev)
        self._run("linear_bn", self.lib.dagr_grid_linear_bn, cells, gs.cnt, xin, cx + 2, lp.b.cout, lp.skipT, lp.sscale,
                  lp.sshift, sk, st)
        out = self._buf(ws, name + "_o", (cells, lp.b.cout), torch.float32, dev)
        self._grid_conv(geom, lv, gs, a, lp.b, sk, out, st)
        return xin, a, out

    def _pool(self, geom, lv_child, gc: GridState, x, aggr, ws, st, dev, keep_temporal):
        """pool level lv_child (0-based) into lv_child+1."""
        lp = lv_child + 1
        child, parent = geom.levels[lv_child], geom.levels[lp]
        gp: GridState = ws["grids"][lp]
        Cc = x.shape[1]
        acc = self._zs(ws, f"acc{lp}", torch.uint8)
        if gp.cells * Cc * 8 > acc.numel():
            raise RuntimeError(f"dagr_b200: pooling accumulator of level {lp + 1} holds {acc.numel()} bytes, {gp.cells * Cc * 8} needed "
                               f"({Cc} channels)")
        accmax = acc.view(torch.int32) if aggr == 0 else None
        accsum = acc.view(torch.float64) if aggr == 1 else None
        possum = self._zs(ws, f"possum{lp}", torch.float64)
        ptmax = self._zs(ws, f"ptmax{lp}", torch.int32)
        pcnt = self._zs(ws, f"pcnt{lp}", torch.int32)
        pmask = self._zs(ws, f"pmask{lp}", torch.int32)
        err = self._zs(ws, "err", torch.int32)
        self._run("grid_pool", self.lib.dagr_grid_pool, child.grid, parent.grid, parent.cellx_dev, parent.celly_dev, gc.cnt,
                  gc.pxy, gc.tmean, gc.tmax, gc.mask, x, Cc, aggr, accmax, accsum, possum, ptmax, pcnt, pmask, err, st)
        gp.x = self._buf(ws, f"gx{lp}", (gp.cells, Cc), torch.float32, dev)
        self._run("grid_pool_finalize", self.lib.dagr_grid_pool_finalize, parent.grid, Cc, aggr, accmax, accsum, possum, ptmax,
                  pcnt, gp.pxy, gp.tmean, gp.tmax, gp.x, st)
        gp.cnt = pcnt[:gp.cells]
        gp.mask = pmask[:gp.cells]
        if keep_temporal:
            self._run("temporal_filter", self.lib.dagr_grid_temporal_filter, parent.grid, gp.cnt, gp.tmax, gp.mask, st)
        return gp

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _append_image(self, geom, lv, gs, o, taps: _Taps, k, ws, st, dev):
        """sampling_skip on a voxel grid (net.py:141-142 etc.): [o | bilinear samples of tap k at the nodes]; o alone for an
        events-only forward."""
        if taps is None:
            return o
        cells, Cc, Cf = gs.cells, o.shape[1], int(taps.feats[k].shape[1])
        xcat = self._buf(ws, f"xcat{lv}", (cells, Cc + Cf), torch.float32, dev)
        xcat[:, :Cc] = o
        pxy = gs.pxy[:cells].long()
        posx = geom.d_posxr[pxy[:, 0]].contiguous()
        posy = geom.d_posyr[pxy[:, 1]].contiguous()
        key = ("bidx", lv)
        if key not in ws:
            per = geom.levels[lv].nx * geom.levels[lv].ny
            ws[key] = (torch.arange(cells, device=dev) // per).int()
        taps.sample_features(self, k, posx, posy, ws[key], cells, geom.W, geom.H, xcat, Cc + Cf, Cc, st)
        return xcat

    @torch.no_grad()
    def forward_events(self, batch_i32: torch.Tensor, pos_i32: torch.Tensor, feat: torch.Tensor, B: int,
                       W: int, H: int, image_feats=None, image_outs=None, stream_state=None, n_old: int = 0, ring=None,
                       image_event=None, ring_streams=None, image_planes=None):
        """batch int32[N], pos int32[N,3], feat fp32[N] (polarity) on CUDA -> decoded [B, A, 5+nc].

        ring = device control block (int32[8], dagr_graph_sort_ring): the three inputs are ring buffers of N = capacity
        slots whose live window {head, count} is only known on the device; every launch then covers the capacity, nothing
        depends on a host-side count and the whole call can sit inside one captured CUDA graph (dagr_b200.streaming).
        ring_streams = S: `ring` is the int32[S+1][8] block of S rings of N / S slots each (dagr_graph_sort_rings), stream s
        being sample s of B = S.
        image_planes = (plane table int32 on the device, stride), with image fusion: image_feats / image_outs are plane arrays
        [P, C, h, w] and sample b reads plane table[b * stride] alone, sampled as a batch of one (the *_planes kernels), so
        each sample gets the bits of a B = 1 forward with its own frame.  The table may be device data written inside the
        step (the stage header, dagr_b200.streaming.FusionMultiStreamDetector).  A plain batch (ring None) takes it too: the
        windows of one recording, each with its own frame (dagr_b200.sequence).
        stream_state, n_old: incremental step (dagr_b200.asynchronous); neither a ring nor image_planes takes it."""
        for n, t in (("batch", batch_i32), ("pos", pos_i32), ("x", feat)):
            _lib.require_cuda(t, n)
        dev = pos_i32.device
        N = int(batch_i32.shape[0])
        mode = resolve_mode(B, N, image_feats, image_outs, stream_state, n_old, ring, ring_streams, image_planes,
                            overlap=self.overlap, profiling=self.prof is not None, use_graphs=self.use_graphs,
                            keep_node_features=self.keep_node_features)
        geom = self.geometry(W, H, B, dev)
        pk = self.pack(geom, dev)
        base = self.workspace(geom, N, dev)
        slot = self._take_slot(mode, dev)
        ws = self._slot_view(base, slot, geom, dev)
        if stream_state is not None:
            stream_state.ensure(geom, N, dev, img_channels=int(image_feats[1].shape[1]) if image_feats is not None else 0)
        kto = bool(getattr(self.model.args, "keep_temporal_ordering", False))
        g1, x1 = self._event_level(mode, geom, pk, ws, N, batch_i32, pos_i32, feat, image_event, kto)
        out, grids, inter, dense_all = self._coarse_stack(mode, slot, geom, pk, ws, g1, B, kto, image_event)
        self.last = dict(geom=geom, ws=ws, N=N, grids=list(grids), inter=inter, dense=dense_all, x1=x1)
        return out

    def _take_slot(self, mode: _Mode, dev) -> int:
        """the hand-off slot of this forward.  An overlapped forward alternates between two and first waits for the last
        coarse stack that read its slot's buffers; a serial one takes slot 0 after every coarse stack in flight."""
        if not mode.overlap:
            self.join()
            return 0
        slot, self._slot = self._slot, self._slot ^ 1
        if self._cstream is None:
            # high priority: the small coarse kernels take SM slots as soon as CTAs of the big event-level kernels retire
            self._cstream = torch.cuda.Stream(device=dev, priority=-1)
        if self._done[slot] is not None:
            torch.cuda.current_stream().wait_event(self._done[slot])
        return slot

    def _cellmask(self, mode: _Mode, ws):
        """the in-edge mask of the pool1 voxels: an incremental call's running mask, else this forward's zeroed one."""
        return mode.state.cellmask if mode.state is not None else self._zs(ws, "cellmask", torch.int32)

    def _event_level(self, mode: _Mode, geom, pk, ws, N, batch_i32, pos_i32, feat, image_event, kto):
        """graph sort -> adjacency + conv_a -> conv_b + pool1 into grid level 0, with the image samples of a hybrid model.
        -> (level-0 grid, the per-event conv_b activations when keep_node_features, else None)"""
        lib, g, st, dev = self.lib, geom.c_geom, _lib.stream_ptr(), pos_i32.device
        taps, state, min_idx = mode.taps, mode.state, mode.min_idx
        ws["zero_buf"].zero_()
        start, perm, ti, xyb, feat_s, nbr, off, xa = (ws[k] for k in ("start", "perm", "ti", "xyb", "feat_s", "nbr", "off", "xa"))
        cellmask = self._cellmask(mode, ws)
        flags = self._zs(ws, "flags", torch.int32)
        wl_hdr = self._zs(ws, "wl_hdr", torch.int32)
        defer = self._dense_policy(ws, wl_hdr, mode.fixed)
        if mode.sort == "rings":
            fn, size = lib.dagr_graph_sort_rings, (N // mode.streams, mode.streams, mode.ring)
        elif mode.sort == "ring":
            fn, size = lib.dagr_graph_sort_ring, (N, mode.ring)
        else:
            fn, size = lib.dagr_graph_sort, (N,)
        self._run("graph_sort", fn, g, batch_i32, pos_i32, feat, *size, ws["key"], ws["tmp"], ws["count"], ws["blocksums"], start,
                  perm, ti, xyb, feat_s, flags, st)
        if min_idx > 0:
            # incremental step: the first n_old arrival indices were processed before; only newer events get their edges /
            # activations computed (the causal graph never changes an old node's inputs), the older xa rows are gathered.
            # With image fusion the frame is the same for every step between two re-seeds (dagr_b200.asynchronous)
            self._run("xa_gather", lib.dagr_xa_permute, N, perm, min_idx, xa, state.xa_arr, 0, st)
        # adjacency + conv_block1.conv_block1.  With image fusion the layer runs on [polarity, 16 image samples, x, y]
        # (net.py:117-126): this is its (polarity, x, y) part, the image channels follow in the conv_a image kernel
        l1a = "l1a" if taps is None else "l1a_img"
        self._run("l1_build", lib.dagr_l1_build_tc, g, N, start, ti, xyb, feat_s, pk[l1a], pk[l1a + "_wfrag"], flags, min_idx,
                  nbr, off, cellmask, xa, wl_hdr, self._zs(ws, "wl_build", torch.int32), defer[0], st)
        skipv = None
        if taps is not None:
            if image_event is not None:                       # stage 1 of the image branch ran on a side stream next to sort + probe
                torch.cuda.current_stream().wait_event(image_event[0])
            x0 = self._buf(ws, "x0img", (2 * max(N, 1) * 8,), torch.float32, dev)
            skipv = self._buf(ws, "skipv", (max(N, 1), 16), torch.float32, dev)
            taps.x0(self, g, N, start, xyb, feat_s, x0, st)
            wl = (wl_hdr[2:], self._zs(ws, "wl_conv_a", torch.int32), defer[1], st)
            if state is not None:
                # only the new nodes are convolved; the xa rows of the older ones are final and stay as gathered
                self._run("l1_conv_a_image_inc", lib.dagr_l1_conv_a_image_inc, g, N, start, xyb, ti, feat_s, x0, nbr, off,
                          pk["l1img"], pk["l1img_wfrag"], min_idx, xa, skipv, *wl)
            else:
                self._run("l1_conv_a_image", lib.dagr_l1_conv_a_image_tc, g, N, start, xyb, feat_s, x0, nbr, off,
                          pk["l1img"], pk["l1img_wfrag"], xa, skipv, *wl)
        if state is not None:
            self._run("xa_scatter", lib.dagr_xa_permute, N, perm, min_idx, xa, state.xa_arr, 1, st)
        x1 = None
        if self.keep_node_features:
            if ws["x1"] is None or ws["x1"].shape[0] < ws["cap"]:
                ws["x1"] = torch.empty((ws["cap"], 16), dtype=torch.float32, device=dev)
            x1 = ws["x1"]
        g1: GridState = ws["grids"][0]
        c1 = 16 + (int(taps.feats[1].shape[1]) if taps is not None else 0)
        g1.x = self._buf(ws, "gx0", (g1.cells, c1), torch.float32, dev)
        self._run("l1_conv_b_pool_voxel", lib.dagr_l1_conv_b_pool_voxel_tc, g, N, start, xyb, ti, feat_s, xa, nbr, off,
                  pk["l1b"], pk["l1b_wfrag"], skipv, min_idx, state.voxmax if state is not None else None, x1, g1.cnt, g1.pxy,
                  g1.tmean, g1.tmax, g1.x, c1, wl_hdr[4:], self._zs(ws, "wl_conv_b", torch.int32), defer[2], st)
        self._dense_report(ws, wl_hdr)
        if taps is not None:
            taps.voxel_max(self, g, N, start, xyb, ti, g1.x, c1, 16, int(pk["l1b"].pool_mean), st)
        g1.mask = cellmask[:g1.cells]
        if kto and state is not None:
            # the persistent stream mask only ever gains edges; the temporal filter (pooling.py:69-72) depends on the CURRENT
            # t_max of both voxels, so it must work on a per-step copy or edges dropped once could never come back
            step_mask = self._zs(ws, "cellmask", torch.int32)
            step_mask[:g1.cells].copy_(cellmask[:g1.cells])
            g1.mask = step_mask[:g1.cells]
        if kto:
            self._run("temporal_filter", lib.dagr_grid_temporal_filter, geom.levels[0].grid, g1.cnt, g1.tmax, g1.mask, st)
        return g1, x1

    def _coarse_stack(self, mode: _Mode, slot, geom, pk, ws, g1, B, kto, image_event):
        """the coarse levels and the head after the event level -> (decoded, grids, layer outputs, dense head maps).  Serial:
        on the caller's stream.  Overlapped: on the side stream once the event level is done; the slot's done-event marks
        the end of its reads, and the results are valid on result_stream()."""
        args = (mode, slot, geom, pk, ws, g1, B, kto, image_event)
        if not mode.overlap:
            res = self._coarse_graph(*args)
            self._out_slot = {}
            return res
        taps = mode.taps
        if taps is not None:                              # the caching allocator must not hand them out while the stack reads
            for t in (*taps.feats, *(t for v in (taps.outs or {}).values() for t in v)):
                t.record_stream(self._cstream)
        fine_done = torch.cuda.Event()
        fine_done.record()
        with torch.cuda.stream(self._cstream):
            self._cstream.wait_event(fine_done)
            res = self._coarse_graph(*args)
            ev = torch.cuda.Event()
            ev.record()
        self._done[slot] = ev
        self._out_slot = {res[0].data_ptr(): slot}
        return res

    def _coarse_graph(self, mode: _Mode, slot, geom, pk, ws, g1, B, kto, image_event):
        """the coarse stack, eager or replayed.  It is ~55 small, fixed-shape launches: replay it as ONE CUDA graph (captured
        on the second call with identical buffers; the event-level kernels stay eager because their grids depend on N).
        With image fusion only the overlapped step is captured (the serial hybrid forward stays eager); its graph reads the
        taps and head maps at fixed addresses, so they and their format are part of the key."""
        args = (mode, geom, pk, ws, g1, B, kto)
        taps = mode.taps
        if not mode.capture:
            return self._coarse(*args, _lib.stream_ptr(), None if image_event is None else image_event[1])
        if image_event is not None:
            # a captured graph cannot wait for an event recorded outside it: the whole stack waits for stage 2
            torch.cuda.current_stream().wait_event(image_event[1])
        gkey = (id(ws.base), slot, self._pack_gen, B, kto, self._cellmask(mode, ws).data_ptr(), bool(self.keep_node_features))
        if taps is not None:
            gkey += (taps.sfx, tuple(t.data_ptr() for t in taps.feats),
                     tuple((k, tuple(t.data_ptr() for t in v)) for k, v in sorted((taps.outs or {}).items())))
        cached = ws.get("graph")
        if cached is not None and cached[0] == gkey:
            cached[1].replay()
            self.launches += cached[3]
            return cached[2]
        l0 = self.launches
        res = self._coarse(*args, _lib.stream_ptr())                 # eager: also allocates every pool buffer
        nk = self.launches - l0
        ws["graph_warm"] = ws.get("graph_warm", 0) + 1
        if ws["graph_warm"] >= 2 and ws.get("graph_key") == gkey:
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            # kernel nodes inherit the priority of the CAPTURE stream: capture on the high-priority side stream in
            # overlap mode so the small coarse kernels get SM slots while a big event-level kernel is resident
            with torch.cuda.graph(gr, stream=self._cstream if mode.overlap else None):
                res_c = self._coarse(*args, _lib.stream_ptr())
            self.launches -= nk                                      # capture enqueues nothing
            ws["graph"] = (gkey, gr, res_c, nk)
        ws["graph_key"] = gkey
        return res

    def _coarse(self, mode: _Mode, geom, pk, ws, g1, B, kto, st, stage2=None):
        """layers 2..5 with their pooling and the head's scales.  stage2: the event on which the image branch's layer2..4
        taps and CNN head maps are ready, waited for after layer2 (eager hybrid forwards)."""
        taps, dev = mode.taps, g1.cnt.device
        aggr = 0 if getattr(self.model.args, "pooling_aggr", "max") == "max" else 1
        lay = pk["layers"]
        _, _, o2 = self._layer(geom, 0, g1, lay[0], ws, "layer2", st, dev)
        if stage2 is not None:
            torch.cuda.current_stream().wait_event(stage2)
        g2 = self._pool(geom, 0, g1, self._append_image(geom, 0, g1, o2, taps, 2, ws, st, dev), aggr, ws, st, dev, kto)
        _, _, o3 = self._layer(geom, 1, g2, lay[1], ws, "layer3", st, dev)
        g3 = self._pool(geom, 1, g2, self._append_image(geom, 1, g2, o3, taps, 3, ws, st, dev), aggr, ws, st, dev, kto)
        _, _, o4 = self._layer(geom, 2, g3, lay[2], ws, "layer4", st, dev)           # out3
        nscale = self.model.head.num_scales
        A = sum(geom.levels[lv].nx * geom.levels[lv].ny for lv in ((2, 3) if nscale == 2 else (3,)))
        out = self._buf(ws, "decoded", (B, A, 5 + self.model.backbone.num_classes), torch.float32, dev)
        dense_all = [None] * nscale
        # The first head scale only needs layer4's output: it runs on a forked stream next to pool4 + layer5 + the second
        # scale (all of them are single-wave kernels on <= B*140 voxels, so they share the GPU instead of queueing);
        # fork / join through events is captured like any other dependency when this stack is replayed as a graph.
        join_ev = None
        if nscale == 2:
            cur = torch.cuda.current_stream()
            if self._fstream is None:
                self._fstream = torch.cuda.Stream(device=dev, priority=-1)
            fork_ev = torch.cuda.Event()
            fork_ev.record(cur)
            with torch.cuda.stream(self._fstream):
                self._fstream.wait_event(fork_ev)
                dense_all[0] = self._head_scale(taps, geom, pk, ws, 0, 2, g3, o4, 0, A, B, out, _lib.stream_ptr())
                join_ev = torch.cuda.Event()
                join_ev.record(self._fstream)
        # pool4 is always mean (net.py:96-97)
        g4 = self._pool(geom, 2, g3, self._append_image(geom, 2, g3, o4, taps, 4, ws, st, dev), 1, ws, st, dev, kto)
        _, _, o5 = self._layer(geom, 3, g4, lay[3], ws, "layer5", st, dev)           # out4
        a0 = geom.levels[2].nx * geom.levels[2].ny if nscale == 2 else 0
        dense_all[nscale - 1] = self._head_scale(taps, geom, pk, ws, nscale - 1, 3, g4, o5, a0, A, B, out, st)
        if join_ev is not None:
            torch.cuda.current_stream().wait_event(join_ev)
        return out, [g1, g2, g3, g4], dict(o2=o2, o3=o3, o4=o4, o5=o5), dense_all

    def _head_scale(self, taps: Optional[_Taps], geom, pk, ws, k, lv, gs: GridState, xo, a0, A, B, out, st):
        """GNNHead.process_feature + collect_outputs + decode_outputs of one scale (dagr.py:179-312) into out[:, a0:].
        -> the dense head maps {cls, reg, obj} of the scale when keep_node_features, else {}"""
        lib, dev, nc = self.lib, gs.cnt.device, self.model.backbone.num_classes
        hp = pk["heads"][k]
        level = geom.levels[lv]
        cells = gs.cells
        nm = f"head{k}"
        stem = self._buf(ws, nm + "_stem", (cells, hp["stem"].cout), torch.float32, dev)
        self._grid_conv(geom, lv, gs, xo, hp["stem"], None, stem, st)
        Cf = hp["cls_conv"].cout
        cr = self._buf(ws, nm + "_cr", (cells, 2 * Cf), torch.float32, dev)          # [cls_feat | reg_feat]
        self._grid_conv(geom, lv, gs, stem, hp["clsreg_conv"], None, cr, st)
        ocls = self._buf(ws, nm + "_cls", (cells, nc), torch.float32, dev)
        self._grid_conv(geom, lv, gs, cr, hp["cls_pred"], None, ocls, st, ldin=2 * Cf)
        oro = self._buf(ws, nm + "_regobj", (cells, 5), torch.float32, dev)         # [reg(4) | obj(1)]
        self._grid_conv(geom, lv, gs, cr[:, Cf:], hp["regobj_pred"], None, oro, st, ldin=2 * Cf)
        form, adds, planes = taps.head_maps(k) if taps is not None else ("", dict.fromkeys(("cls", "reg", "obj")), ())
        self._run("head_finish", getattr(lib, "dagr_head_finish" + form), level.grid, gs.cnt, ocls, nc, oro, 5, adds["cls"],
                  adds["reg"], adds["obj"], nc, int(self.model.backbone.strides[k]), a0, A, *planes, out, st)
        dense = {}
        if self.keep_node_features:
            # parity / debugging: the dense [B,C,ny,nx] head maps of SplineConvToDense (spline_conv.py:80-107)
            for name, src, c0, cw, ld in (("cls", ocls, 0, nc, nc), ("reg", oro, 0, 4, 5), ("obj", oro, 4, 1, 5)):
                d = self._buf(ws, nm + "_d" + name, (B, cw, level.ny, level.nx), torch.float32, dev)
                self._run("to_dense", lib.dagr_grid_to_dense, level.grid, gs.cnt, src[:, c0:], cw, ld, adds[name], d, st)
                dense[name] = d
        return dense

    def xa_rows(self):
        """conv_block1.conv_block1 activations of the last forward as [N,16] rows in sorted order
        (the kernels keep them half-major, [2][N][8])."""
        L = self.last
        N, xa = L["N"], L["ws"]["xa"]
        rows = torch.cat([xa[:N * 8].view(N, 8), xa[N * 8:2 * N * 8].view(N, 8)], dim=1).clone()
        sw = ((torch.arange(N, device=rows.device) >> 2) & 1).bool()       # XA_SWZ: 16-byte chunks swapped on these rows
        r = rows[sw].view(-1, 2, 2, 4)
        rows[sw] = r.flip(2).reshape(-1, 16)
        return rows

    @torch.no_grad()
    def postprocess(self, decoded: torch.Tensor, conf_thre, nms_thre, width, height, filtering=True):
        """postprocess_network_output on device (model/utils.py:61-110): det [B,A,6], ndet [B]."""
        B, A, D = decoded.shape
        nc = D - 5
        dev = decoded.device
        slot = self._out_slot.get(decoded.data_ptr()) if self.overlap else None
        if slot is None:
            det = torch.empty((B, A, 6), dtype=torch.float32, device=dev)
            ndet = torch.empty(B, dtype=torch.int32, device=dev)
            self._run("postprocess_nms", self.lib.dagr_postprocess_nms, decoded, B, A, nc, float(conf_thre), float(nms_thre),
                      int(width), int(height), 1 if filtering else 0, det, ndet, _lib.stream_ptr())
            return det, ndet
        # overlapped forward: NMS follows the coarse stack on the side stream, into per-slot result buffers
        sw = self.last["ws"]
        det = self._buf(sw, "post_det", (B, A, 6), torch.float32, dev)
        ndet = self._buf(sw, "post_ndet", (B,), torch.int32, dev)
        with torch.cuda.stream(self._cstream):
            self._run("postprocess_nms", self.lib.dagr_postprocess_nms, decoded, B, A, nc, float(conf_thre), float(nms_thre),
                      int(width), int(height), 1 if filtering else 0, det, ndet, _lib.stream_ptr())
            ev = torch.cuda.Event()
            ev.record()
        self._done[slot] = ev
        return det, ndet

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def export_edges(self):
        """edge_index int64[2,E] in the reference's layout for the last forward (host sync)."""
        L = self.last
        geom, ws, N = L["geom"], L["ws"], L["N"]
        dev = ws["perm"].device
        if N == 0:
            return torch.zeros((2, 0), dtype=torch.long, device=dev)
        cap = geom.K * N
        inv = torch.empty(N, dtype=torch.int32, device=dev)
        rowptr = torch.empty(N + 1, dtype=torch.int32, device=dev)
        es = torch.empty(cap, dtype=torch.int64, device=dev)
        ed = torch.empty(cap, dtype=torch.int64, device=dev)
        self._run("graph_export", self.lib.dagr_graph_export, geom.c_geom, N, ws["perm"], ws["ti"], ws["nbr"], inv, rowptr,
                  ws["blocksums"], es, ed, cap, _lib.stream_ptr())
        E = int(rowptr[N].item())
        return torch.stack([es[:E], ed[:E]])
