"""The dense image branch of the hybrid detector -- ResNet trunk taps (`HookModule`, reference
src/dagr/model/networks/net_img.py:42-135), nearest resize of the two output taps and the YOLOX-style `CNNHead`
(dagr.py:106-122,205-206) -- as TWO replayed CUDA graphs on a side stream.

The branch does not depend on the events, so it runs concurrently with the graph kernels of the same forward:
  stage 1 (conv1 .. layer1 + their 1x1 tap convs) next to the cell-major sort and the radius-graph probe; the event-level
          convs wait for its event (they sample the conv1 / layer1 taps);
  stage 2 (layer2 .. layer4, remaining tap convs, resize, CNN head) next to the event-level convs (latency-bound fp32 SIMT
          kernels at ~30 % occupancy, while the trunk is tensor-core work); the coarse stack waits for its event.
Arithmetic is untouched: the same torch modules run (cuDNN, TF32 convolutions like the reference's default), only captured
once per input shape instead of ~250 eager launches per forward -- at batch 1 the eager trunk is bound by host launch
time, not by the GPU (SURVEY 8(f) rank 3).

precision "bf16" (DAGR.image_precision) runs a bf16, channels_last copy of backbone.net and head.cnn_head that the branch
owns, under torch.autocast(bfloat16); the model's own fp32 modules are never converted, so "tf32" keeps its bits.  The copy
follows the weights: it is rebuilt when Engine._params_key changes and on invalidate() (load_state_dict, .to()).  Its five
feature taps stay bf16 NHWC (channels_last [B, C, h, w]), which the engine's bf16 sampling kernels read; the CNN head maps are
converted to fp32 NCHW inside the graph.  The input is the formatted fp32 image in both precisions.  Graphs are keyed by
(shape, device, precision), so a model used in both keeps both sets.
"""
from __future__ import annotations

import copy

import torch

PRECISIONS = ("tf32", "bf16")


def _bf16_copy(module):
    """a channels_last copy of `module` whose convolutions hold bf16 weights (autocast then casts nothing per call); the
    batch norms keep fp32 parameters and statistics, as autocast would use them."""
    m = copy.deepcopy(module).to(memory_format=torch.channels_last)
    for c in m.modules():
        if isinstance(c, torch.nn.Conv2d):
            c.to(torch.bfloat16)
    return m


class ImageBranch:
    def __init__(self, model):
        self.model = model
        self.stream = None
        self._sizes = None         # head grid sizes: read once (a device->host read is not allowed under graph capture)
        self._graphs = {}          # (shape, device, precision) -> dict(g1, g2, inp, mid, feats, outs, warm)
        self._bf16 = None          # (weights key, bf16 copy of backbone.net, bf16 copy of head.cnn_head)

    def invalidate(self):
        self._graphs = {}
        self._bf16 = None

    def _refresh_bf16(self):
        """make the bf16 copy current: rebuilt when the weights changed (its graphs hold the old copy's parameters and go
        with it)."""
        m = self.model
        key = m.engine._params_key()
        if self._bf16 is None or self._bf16[0] != key:
            self._graphs = {k: v for k, v in self._graphs.items() if k[2] != "bf16"}
            self._bf16 = (key, _bf16_copy(m.backbone.net), _bf16_copy(m.head.cnn_head))

    def _stage1(self, image, precision):
        """precision "bf16" runs the copy that _refresh_bf16() made current"""
        if precision == "tf32":
            taps, mid = self.model.backbone.net.stage1(image)
            return [t.float().contiguous() for t in taps], mid
        with torch.autocast("cuda", dtype=torch.bfloat16):
            taps, mid = self._bf16[1].stage1(image.contiguous(memory_format=torch.channels_last))
        return [t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last) for t in taps], mid

    def _stage2(self, mid, precision):
        m = self.model
        if precision == "tf32":
            feats, image_outs = self._head(m.backbone.net, m.head.cnn_head, mid)
            feats = [f.float().contiguous() for f in feats]
        else:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                feats, image_outs = self._head(self._bf16[1], self._bf16[2], mid)
            feats = [f.to(torch.bfloat16).contiguous(memory_format=torch.channels_last) for f in feats]
        return feats, {k: [t.float().contiguous() for t in v] for k, v in image_outs.items()}

    def _head(self, net, cnn_head, mid):
        m = self.model
        feats, outs = net.stage2(mid)
        if self._sizes is None:
            self._sizes = m.backbone.get_output_sizes()[-m.head.num_scales:]
        cnn_in = [torch.nn.functional.interpolate(o, size=tuple(sz)) for o, sz in zip(outs[-m.head.num_scales:], self._sizes)]
        return feats, cnn_head(cnn_in)

    @torch.no_grad()
    def run(self, image: torch.Tensor, use_graph: bool = True, precision: str = "tf32"):
        """-> (image_feats, image_outs, (event1, event2)): the first two feature maps are valid on any stream that waited
        for event1, everything else after event2; all of them are overwritten by the next call (static graph buffers).
        precision "tf32": fp32 NCHW feature maps; "bf16": bf16 channels_last ones (the module docstring)."""
        if precision not in PRECISIONS:
            raise ValueError(f"image precision {precision!r}: expected one of {PRECISIONS}")
        dev = image.device
        cur = torch.cuda.current_stream(dev)
        if self.stream is None:
            self.stream = torch.cuda.Stream(device=dev)
        s = self.stream
        s.wait_stream(cur)                                   # the image is ready and every consumer of the previous outputs is done
        if precision == "bf16":
            self._refresh_bf16()                             # before its graphs are looked up
        key = (tuple(image.shape), str(dev), precision)
        st = self._graphs.get(key)
        with torch.cuda.stream(s):
            ev1, ev2 = torch.cuda.Event(), torch.cuda.Event()
            if not use_graph:
                f12, mid = self._stage1(image.float(), precision)
                ev1.record(s)
                f345, outs = self._stage2(mid, precision)
            elif st is None or st.get("g1") is None:
                if st is None:
                    st = dict(g1=None, inp=torch.empty(image.shape, dtype=torch.float32, device=dev), warm=0)
                    self._graphs[key] = st
                st["inp"].copy_(image)
                f12, mid = self._stage1(st["inp"], precision)  # eager warm-up (cuDNN algorithm selection, workspaces)
                ev1.record(s)
                f345, outs = self._stage2(mid, precision)
                st["warm"] += 1
                if st["warm"] >= 2:
                    s.synchronize()
                    g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g1, stream=s):
                        gf12, gmid = self._stage1(st["inp"], precision)
                    with torch.cuda.graph(g2, stream=s, pool=g1.pool()):
                        gf345, gouts = self._stage2(gmid, precision)
                    st.update(g1=g1, g2=g2, f12=gf12, f345=gf345, outs=gouts)
                    g1.replay()                              # fill the static outputs for this call
                    ev1 = torch.cuda.Event()
                    ev1.record(s)
                    g2.replay()
                    f12, f345, outs = gf12, gf345, gouts
            else:
                st["inp"].copy_(image)
                st["g1"].replay()
                ev1.record(s)
                st["g2"].replay()
                f12, f345, outs = st["f12"], st["f345"], st["outs"]
            ev2.record(s)
        feats = list(f12) + list(f345)
        for t in feats:
            t.record_stream(cur)
        for v in outs.values():
            for t in v:
                t.record_stream(cur)
        return feats, outs, (ev1, ev2)
