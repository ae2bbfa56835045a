"""oracle/ref_ops.py -- TEST INFRASTRUCTURE ONLY.

CPU (torch fp32 / int64) restatement of every op on DAGR's hot path, following the
reference op for op.  Nothing in the product (`dagr_b200/`) may import this module;
only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg do.

Pinning status
--------------
* graph build (`RefGraph`): wraps oracle/graph_oracle.c, which is cross-checked on the
  GPU box against the reference's own CUDA kernels compiled into oracle/_ref/ -> PINNED.
* everything else restates third-party packages that are NOT vendored in the reference
  and not installable offline (torch_geometric ~2.0.x, torch_spline_conv ~1.2.1,
  torch_scatter ~2.0.9, torch_cluster ~1.6.0, torch_sparse ~0.6.13, YOLOX @618fd8c0;
  install_env.sh:7-11, download_and_install_dependencies.sh:15).  Their published
  algorithms are restated below and anchored on the reference's call sites; the only
  known-answer vectors are the self-consistent KATs in tests/golden/spline_kats.json.
  -> PARITY UNPINNED for those ops (no golden vectors exist in the reference).
"""
from __future__ import annotations

import ctypes
import math
import os
from pathlib import Path
from typing import List, Optional, Tuple

import numpy as np
import torch

_HERE = Path(__file__).resolve().parent


# ----------------------------------------------------------------------------------------
# graph build  (src/dagr/graph/ev_graph.py:18-166, graph/utils.py:6-23, ev_graph.cu, spiral.h)
# ----------------------------------------------------------------------------------------
def _load_graph_lib():
    so = _HERE / "libgraph_oracle.so"
    if not so.exists():
        import subprocess
        subprocess.check_call(["make", "-C", str(_HERE), "libgraph_oracle.so"])
    lib = ctypes.CDLL(str(so))
    lib.graph_oracle_create.restype = ctypes.c_void_p
    lib.graph_oracle_create.argtypes = [ctypes.c_int] * 4
    lib.graph_oracle_destroy.argtypes = [ctypes.c_void_p]
    lib.graph_oracle_reset.argtypes = [ctypes.c_void_p]
    lib.graph_oracle_delete_nodes.argtypes = [ctypes.c_void_p, ctypes.c_int64]
    lib.graph_oracle_num_nodes.restype = ctypes.c_int64
    lib.graph_oracle_num_nodes.argtypes = [ctypes.c_void_p]
    lib.graph_oracle_forward.restype = ctypes.c_int64
    lib.graph_oracle_forward.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                         ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


_GLIB = None


class RefGraph:
    """SlidingWindowGraph restated (ev_graph.py:106-166) on top of graph_oracle.c."""

    def __init__(self, width, height, batch_size=1, max_num_neighbors=16, max_queue_size=128,
                 radius=7, delta_t_us=10000):
        global _GLIB
        if _GLIB is None:
            _GLIB = _load_graph_lib()
        self.lib = _GLIB
        self.W, self.H, self.B = int(width), int(height), int(batch_size)
        self.K, self.Q = int(max_num_neighbors), int(max_queue_size)
        self.radius, self.delta_t_us = int(radius), int(delta_t_us)
        self.h = self.lib.graph_oracle_create(self.B, self.Q, self.H, self.W)
        if not self.h:
            raise MemoryError("graph oracle allocation failed")
        self.edges = torch.zeros((2, 0), dtype=torch.long)

    def __del__(self):
        try:
            self.lib.graph_oracle_destroy(self.h)
        except Exception:
            pass

    def reset(self):
        self.lib.graph_oracle_reset(self.h)
        self.edges = torch.zeros((2, 0), dtype=torch.long)

    @property
    def init(self):
        return self.lib.graph_oracle_num_nodes(self.h) > 0

    def delete_nodes(self, n_delete):                     # ev_graph.py:121-136
        self.lib.graph_oracle_delete_nodes(self.h, int(n_delete))
        mask = (self.edges[0] < n_delete) | (self.edges[1] < n_delete)
        deleted = self.edges[:, mask].clone()
        self.edges = self.edges[:, ~mask] - n_delete
        return deleted

    def forward(self, batch: torch.Tensor, pos: torch.Tensor, delete_nodes=False, collect_edges=True):
        """batch int32[N], pos int32[N,3] -> edge_index int64[2,E] (ev_graph.py:139-166)."""
        n_delete = len(batch) if self.init else 0
        N = int(batch.shape[0])
        if N == 0:
            return torch.zeros((2, 0), dtype=torch.long)
        b = np.ascontiguousarray(batch.cpu().numpy().astype(np.int32))
        p = np.ascontiguousarray(pos.cpu().numpy().astype(np.int32))
        src = np.empty(self.K * N, dtype=np.int64)
        dst = np.empty(self.K * N, dtype=np.int64)
        E = self.lib.graph_oracle_forward(self.h, b.ctypes.data, p.ctypes.data, N, self.K, self.radius,
                                          self.delta_t_us, src.ctypes.data, dst.ctypes.data)
        if E < 0:
            raise RuntimeError("graph oracle failed")
        edges = torch.from_numpy(np.stack([src[:E], dst[:E]]))
        if collect_edges:
            self.edges = torch.cat([self.edges, edges], dim=-1)
        if delete_nodes:
            self.delete_nodes(n_delete)
        return edges


def denormalize_pos(pos: torch.Tensor, width: int, height: int, time_window: int) -> torch.Tensor:
    """src/dagr/model/layers/ev_tgn.py:11-16."""
    denorm = torch.tensor([int(width), int(height), int(time_window)])
    return (denorm.view(1, -1) * pos + 1e-3).int()


def format_pos(xy: torch.Tensor, t: torch.Tensor, width: int, height: int, time_window: int) -> torch.Tensor:
    """src/dagr/utils/buffers.py:33-44 (pos part): int -> fp32 true division."""
    normalizer = torch.stack([torch.tensor(width), torch.tensor(height), torch.tensor(time_window)], dim=-1)
    pos = torch.cat([xy, t.view(-1, 1)], dim=-1)
    return pos / normalizer


# ----------------------------------------------------------------------------------------
# edge attributes (PyG T.Cartesian; restated in-repo at src/dagr/asynchronous/cartesian.py:6-16)
# ----------------------------------------------------------------------------------------
def cartesian(pos: torch.Tensor, edge_index: torch.Tensor, max_value: float) -> torch.Tensor:
    if edge_index.shape[1] == 0:                                   # components.py:31-35
        return torch.zeros((0, pos.shape[1]), dtype=pos.dtype)
    row, col = edge_index
    cart = pos[row] - pos[col]
    return cart / (2 * max_value) + 0.5


# ----------------------------------------------------------------------------------------
# torch_spline_conv.spline_basis / spline_weighting  (published algorithm, degree 1)
# ----------------------------------------------------------------------------------------
def spline_basis(pseudo: torch.Tensor, kernel_size: int = 5, is_open: bool = True, degree: int = 1):
    """basis[E, 2^dim], weight_index[E, 2^dim] for degree-1 B-splines.

    for s in 0..2^dim-1: k_d = (s >> d) & 1; v = pseudo_d * (ks - degree*open);
      index += ((int)v + k_d) % ks * ks^d ; frac = v - floor(v); basis *= k_d ? frac : 1-frac
    """
    assert degree == 1
    E, dim = pseudo.shape
    S = 2 ** dim
    basis = torch.ones((E, S), dtype=pseudo.dtype)
    index = torch.zeros((E, S), dtype=torch.long)
    offset = 1
    for d in range(dim):
        v = pseudo[:, d] * float(kernel_size - degree * int(is_open))
        fl = torch.floor(v)
        frac = v - fl
        for s in range(S):
            k = (s >> d) & 1
            index[:, s] += ((v.to(torch.long) + k) % kernel_size) * offset
            basis[:, s] = basis[:, s] * (frac if k == 1 else (1 - frac))
        offset *= kernel_size
    return basis, index


def spline_weighting(x_j: torch.Tensor, weight: torch.Tensor, basis: torch.Tensor, index: torch.Tensor):
    """out[e,o] = sum_s basis[e,s] * sum_i x[e,i] * W[index[e,s], i, o]   (s outer, i inner)."""
    E = x_j.shape[0]
    out = torch.zeros((E, weight.shape[2]), dtype=x_j.dtype)
    for s in range(basis.shape[1]):
        w = weight[index[:, s]]                       # [E, Cin, Cout]
        out = out + basis[:, s:s + 1] * torch.einsum("ei,eio->eo", x_j, w)
    return out


def lut_params_layer1(radius: float, width: int):
    """DAGR.cache_luts for the event level (src/dagr/model/networks/dagr.py:38-41)."""
    M = 2 * float(int(radius * width + 2) / width)
    r = int(radius * width + 1)
    return r, r, M


def build_lut(weight: torch.Tensor, height: int, width: int, rx: int, Mx: float, ry=None, My=None, kernel_size=5):
    """MySplineConv.init_lut (src/dagr/model/layers/spline_conv.py:16-37)."""
    ry = ry or rx
    My = My or Mx
    remap = torch.Tensor([[2 * Mx * width, 0, -Mx * width + rx],
                          [0, 2 * My * height, -My * height + ry]])
    dxy = torch.stack(torch.meshgrid(torch.arange(-rx, rx + 1), torch.arange(-ry, ry + 1), indexing="ij")).float()
    dxy[0] = dxy[0] / (2 * Mx * width) + 0.5
    dxy[1] = dxy[1] / (2 * My * height) + 0.5
    edge_attr = dxy.view((2, -1)).t()
    bil_w, indices = spline_basis(edge_attr, kernel_size, True, 1)
    lut = (bil_w[..., None, None] * weight[indices]).sum(1)
    _, cin, cout = lut.shape
    return lut.view((2 * rx + 1, 2 * ry + 1, cin, cout)), remap


def message_lut(x_j, edge_attr, lut, remap):
    """MySplineConv.message_lut (spline_conv.py:39-47)."""
    dx = (edge_attr[:, 0] * remap[0, 0] + remap[0, -1] + 1e-3).long()
    dy = (edge_attr[:, 1] * remap[1, 1] + remap[1, -1] + 1e-3).long()
    w = lut[dx, dy]
    return torch.einsum("nio,ni->no", w, x_j)


CHUNK_ELEMS = 64_000_000     # floats per [E,Cin,Cout] temporary


def to_sparse(edge_index: torch.Tensor, edge_attr: torch.Tensor, N: int):
    """PyG ToSparseTensor: stable sort of edges (and attrs) by key dst*N + src; CSR over dst."""
    row, col = edge_index
    key = col * N + row
    perm = torch.argsort(key, stable=True)
    return row[perm], col[perm], edge_attr[perm]


def spline_conv(x: torch.Tensor, edge_index: torch.Tensor, edge_attr: torch.Tensor, weight: torch.Tensor,
                root: torch.Tensor, bias: Optional[torch.Tensor] = None, lut=None, remap=None,
                kernel_size: int = 5) -> torch.Tensor:
    """MySplineConv.forward/_forward (spline_conv.py:49-78) incl. PyG propagate + segment_csr(sum).

    weight [25,Cin,Cout]; root = lin.weight [Cout,Cin]; messages are summed per destination in the
    (dst, src)-sorted order, sequentially (index_add_ on CPU is sequential).
    """
    N = x.shape[0]
    out = torch.zeros((N, weight.shape[2]), dtype=x.dtype)
    if edge_index.numel() > 0:                                      # spline_conv.py:67-70
        attr = edge_attr[:, :2]
        src, dst, attr = to_sparse(edge_index, attr, N)
        E = src.shape[0]
        # edges are processed in chunks only to bound the [E,Cin,Cout] temporary (the reference
        # materialises it in one go, spline_conv.py:44); per-destination order is unchanged
        step = max(1, int(CHUNK_ELEMS // max(1, weight.shape[1] * weight.shape[2])))
        for s0 in range(0, E, step):
            sl = slice(s0, min(E, s0 + step))
            x_j = x[src[sl]]
            if lut is not None:
                msg = message_lut(x_j, attr[sl], lut, remap)
            else:
                basis, index = spline_basis(attr[sl], kernel_size, True, 1)
                msg = spline_weighting(x_j, weight, basis, index)
            out.index_add_(0, dst[sl], msg)
    out = out + x @ root.t()                                        # :72-73
    if bias is not None:
        out = out + bias                                            # :75-76
    return out


def batch_norm_eval(x, weight, bias, mean, var, eps=1e-5):
    """PyG BatchNorm == torch.nn.BatchNorm1d(eps=1e-5) in eval mode (components.py:9-12)."""
    return torch.nn.functional.batch_norm(x, mean, var, weight, bias, False, 0.1, eps)


# ----------------------------------------------------------------------------------------
# pooling (src/dagr/model/layers/pooling.py:12-97 + torch_cluster.grid_cluster + torch_scatter)
# ----------------------------------------------------------------------------------------
def compute_pooling_at_each_layer(pooling_dim_at_output: str, num_layers: int = 4) -> torch.Tensor:
    """src/dagr/model/networks/net.py:19-28."""
    py, px = map(int, pooling_dim_at_output.split("x"))
    base = torch.tensor([1.0 / px, 1.0 / py, 1.0 / 1])
    out = []
    for i in range(num_layers):
        p = base / 2 ** (3 - i)
        p[-1] = 1
        out.append(p)
    return torch.stack(out)


def grid_cluster(pos: torch.Tensor, size: torch.Tensor, start: torch.Tensor, end: torch.Tensor) -> torch.Tensor:
    """torch_cluster.grid_cluster: c = sum_d (int64)((pos_d-start_d)/size_d) * k_d,
    k = exclusive cumprod of ((int64)((end_d-start_d)/size_d) + 1)   (fp32 IEEE division, C-cast)."""
    pos = pos - start.unsqueeze(0)
    num_voxels = ((end - start) / size).to(torch.long) + 1
    num_voxels = num_voxels.cumprod(0)
    num_voxels = torch.cat([torch.ones(1, dtype=torch.long), num_voxels], 0)[: size.shape[0]]
    out = (pos / size.view(1, -1)).to(torch.long)
    out = out * num_voxels.view(1, -1)
    return out.sum(1)


def consecutive_cluster(src: torch.Tensor):
    """pooling.py:12-16 (perm picks *some* member; the last write wins on CPU)."""
    unique, inv, counts = torch.unique(src, sorted=True, return_inverse=True, return_counts=True)
    perm = torch.arange(inv.size(0), dtype=inv.dtype)
    perm = inv.new_empty(unique.size(0)).scatter_(0, inv, perm)
    return unique, inv, perm, counts


def scatter_mean(x: torch.Tensor, index: torch.Tensor, n: int):
    out = torch.zeros((n,) + x.shape[1:], dtype=x.dtype)
    out.index_add_(0, index, x)
    cnt = torch.zeros(n, dtype=x.dtype)
    cnt.index_add_(0, index, torch.ones(index.shape[0], dtype=x.dtype))
    cnt = cnt.clamp(min=1)
    return out / cnt.view(-1, *([1] * (x.dim() - 1)))


def scatter_max(x: torch.Tensor, index: torch.Tensor, n: int):
    out = torch.full((n,) + x.shape[1:], float("-inf"), dtype=x.dtype)
    idx = index.view(-1, *([1] * (x.dim() - 1))).expand_as(x)
    out = out.scatter_reduce(0, idx, x, reduce="amax", include_self=True)
    return out


def round_to_pixel(pos: torch.Tensor, wh_inv: torch.Tensor):
    """pooling.py:47-49."""
    q = torch.div(pos + 1e-5, wh_inv, rounding_mode="floor")
    return q * wh_inv


def pooling(x, pos, batch, edge_index, voxel_size3, width, height, batch_size, cart_max, aggr="max",
            keep_temporal_ordering=False, exact_mean=True, pos_hint=None, mirror_t_quirk=True):
    """Pooling.forward (pooling.py:51-97).  Returns dict(x,pos,batch,edge_index,edge_attr,cluster,ambiguous).

    `exact_mean`: the reference's pooled position is an fp32 atomic mean (run-to-run unstable);
    the oracle computes it in float64 and flags clusters whose pixel rounding is within float
    noise of a boundary (`ambiguous`), see SURVEY H3(b).
    `pos_hint` (fp32 [n,2], optional): rounded positions to adopt for the clusters the oracle itself flags as
    ambiguous, so that a comparison can continue below such a voxel instead of stopping (the reference is not
    run-to-run stable there).  `mirror_t_quirk=False` keeps an event with normalised t == 1.0 (dsec_data.py:145)
    in temporal cell 0 instead of letting it alias into the next sample's voxel (SURVEY quirk Q1 / H3a).
    """
    if x.shape[0] == 0:
        return None
    voxel_size = torch.cat([voxel_size3, torch.Tensor([1])])                    # pooling.py:24
    start = torch.Tensor([0, 0, 0, 0])
    end = torch.Tensor([0.9999999, 0.9999999, 0.9999999, batch_size - 1])     # :31
    wh_inv = 1 / torch.Tensor([[width, height]])                               # :32
    pos4 = torch.cat([pos, batch.float().view(-1, 1)], dim=-1)                 # :55
    if not mirror_t_quirk:
        pos4[:, 2] = pos4[:, 2].clamp(max=0.9999999)
    cluster = grid_cluster(pos4, voxel_size, start, end)                       # :56
    uniq, cl, perm, _ = consecutive_cluster(cluster)                            # :57
    n = uniq.shape[0]
    ei = cl[edge_index]                                                         # :58
    ei = ei[:, ei[0] != ei[1]]                                                  # :62
    if ei.shape[1] > 0:
        ei = ei.unique(dim=-1)                                                  # :64
    nbatch = batch[perm]                                                        # :66
    if exact_mean:
        npos64 = scatter_mean(pos.double(), cl, n)
        npos = npos64.float()
    else:
        npos = scatter_mean(pos, cl, n)                                         # :67 pool_pos
        npos64 = npos.double()
    if keep_temporal_ordering:                                                  # :69-72
        t_max = scatter_max(pos[:, -1], cl, n)
        ei = ei[:, t_max[ei[1]] > t_max[ei[0]]]
    if aggr == "max":
        nx = scatter_max(x, cl, n)                                              # :75
    else:
        nx = scatter_mean(x, cl, n)                                             # :77
    # ambiguity: distance of (mean+1e-5)*W to the next integer boundary, in pixels
    scaled = (npos64[:, :2] + 1e-5) * torch.tensor([width, height], dtype=torch.float64)
    frac = scaled - torch.floor(scaled)
    ambiguous = ((frac < 2e-3) | (frac > 1 - 2e-3)).any(dim=1)
    npos = npos.clone()
    npos[:, :2] = round_to_pixel(npos[:, :2], wh_inv)                           # :86
    if pos_hint is not None and bool(ambiguous.any()) and pos_hint.shape[0] == n:
        npos[ambiguous, :2] = pos_hint[ambiguous].to(npos.dtype)
    edge_attr = cartesian(npos, ei, cart_max) if ei.shape[1] > 0 else torch.zeros((0, npos.shape[1]))
    return dict(x=nx, pos=npos, batch=nbatch, edge_index=ei, edge_attr=edge_attr, cluster=cl,
                unique_clusters=uniq, ambiguous=ambiguous)


# ----------------------------------------------------------------------------------------
# dense projection, decode, post-process
# ----------------------------------------------------------------------------------------
def to_dense(x, pos, pooling3, batch, batch_size):
    """spline_conv.py:80-107."""
    Wg, Hg = (1 / pooling3[:2] + 1e-3).long()
    C = x.shape[-1]
    dense = torch.zeros((batch_size, C, int(Hg), int(Wg)), dtype=x.dtype)
    est_x, est_y = (pos[:, :2] / pooling3[:2]).t().long()
    dense[batch.long(), :, est_y, est_x] = x
    return dense


def init_grid_and_stride(hw, strides):
    """src/dagr/model/utils.py:119-132."""
    grids, all_strides = [], []
    for (hsize, wsize), stride in zip(hw, strides):
        yv, xv = torch.meshgrid(torch.arange(hsize), torch.arange(wsize), indexing="ij")
        grid = torch.stack((xv, yv), 2).view(1, -1, 2)
        grids.append(grid)
        all_strides.append(torch.full((*grid.shape[:2], 1), stride))
    return torch.cat(grids, dim=1).float(), torch.cat(all_strides, dim=1).float()


def decode_outputs(outputs, hw, strides):
    """GNNHead.decode_outputs (dagr.py:306-312)."""
    grid, stride = init_grid_and_stride(hw, strides)
    outputs = outputs.clone()
    outputs[..., :2] = (outputs[..., :2] + grid) * stride
    outputs[..., 2:4] = torch.exp(outputs[..., 2:4]) * stride
    return outputs


def box_iou_one_to_many(box, boxes):
    x1 = torch.maximum(box[0], boxes[:, 0]); y1 = torch.maximum(box[1], boxes[:, 1])
    x2 = torch.minimum(box[2], boxes[:, 2]); y2 = torch.minimum(box[3], boxes[:, 3])
    inter = (x2 - x1).clamp(min=0) * (y2 - y1).clamp(min=0)
    a = (box[2] - box[0]) * (box[3] - box[1])
    b = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    return inter / (a + b - inter)


def nms(boxes, scores, thr):
    """torchvision.ops.nms semantics: descending score, suppress IoU > thr."""
    order = torch.argsort(scores, descending=True, stable=True)
    keep = []
    suppressed = torch.zeros(len(order), dtype=torch.bool)
    for ii in range(len(order)):
        if suppressed[ii]:
            continue
        i = order[ii]
        keep.append(int(i))
        if ii + 1 < len(order):
            rest = order[ii + 1:]
            iou = box_iou_one_to_many(boxes[i], boxes[rest])
            suppressed[ii + 1:] |= iou > thr
    return torch.tensor(keep, dtype=torch.long)


def postprocess_network_output(prediction, num_classes, conf_thre=0.001, nms_thre=0.65, height=480, width=640,
                               filtering=True):
    """src/dagr/model/utils.py:61-110 (incl. the obj*cls^2 confidence quirk, :80-82)."""
    prediction = prediction.clone()
    prediction[..., :2] -= prediction[..., 2:4] / 2
    prediction[..., 2:4] += prediction[..., :2]
    output = []
    for image_pred in prediction:
        class_conf, class_pred = torch.max(image_pred[:, 5:5 + num_classes], 1, keepdim=True)
        image_pred[:, 4:5] *= class_conf
        conf_mask = (image_pred[:, 4] * class_conf.squeeze(1) >= conf_thre)
        det = torch.cat((image_pred[:, :5], class_pred.float()), 1)
        if filtering:
            det = det[conf_mask]
        if len(det) == 0:
            output.append(dict(boxes=torch.zeros(0, 4), scores=torch.zeros(0), labels=torch.zeros(0, dtype=torch.long)))
            continue
        max_dim = max(width, height)
        offs = det[:, 5] * float(max_dim + 1)                      # utils.py:25-33
        keep = nms(det[:, :4] + offs[:, None], det[:, 4], nms_thre)
        if filtering:
            det = det[keep]
        output.append(dict(boxes=det[:, :4], scores=det[:, 4], labels=det[:, -1].long()))
    return output


# ----------------------------------------------------------------------------------------
# image feature sampling (src/dagr/model/networks/net.py:193-221)
# ----------------------------------------------------------------------------------------
def sample_features(pos, batch, image_feat, width, height, mode="bilinear"):
    x = pos[:, 0] * width
    y = pos[:, 1] * height
    b = batch.float()
    batch_size = image_feat.shape[0]
    x = 2 * x / (width - 1) - 1
    y = 2 * y / (height - 1) - 1
    bs = batch_size if batch_size > 1 else 2
    b = 2 * b / (bs - 1) - 1
    grid = torch.stack((x, y, b), dim=-1).view(1, 1, 1, -1, 3)
    feat = image_feat.permute(1, 0, 2, 3).unsqueeze(0)
    out = torch.nn.functional.grid_sample(feat, grid=grid, mode=mode, align_corners=True)
    return out.view(feat.shape[1], -1).t()


# ----------------------------------------------------------------------------------------
# asy_tools (src/dagr/asynchronous/asy_tools/main.cu)
# ----------------------------------------------------------------------------------------
def masked_isdiff(indices, x_old, x_new, atol, rtol):
    """main.cu:14-41,97-125: keeps r where any_c |old-new| > atol + rtol*new (signed new)."""
    keep = []
    for r in indices.tolist():
        a, b = x_old[r], x_new[r]
        if bool(((a - b).abs() > atol + rtol * b).any()):
            keep.append(r)
    return torch.tensor(keep, dtype=torch.long)


def masked_inplace_bn(indices, x, x_out, mean, var, weight, bias, eps):
    """main.cu:43-67.  nvcc contracts `* weight + bias` there to one fma.rn, so d * w + b is rounded once: the product of
    two float32 values is exact in float64, and the float64 sum is cast to float32."""
    r = indices.long()
    d = (x[r] - mean) / torch.sqrt(var + eps)
    x_out[r] = (d.double() * weight.double() + bias.double()).to(x_out.dtype)
    return x_out


def masked_lin(indices, x_in, x_out, weight, bias=None, add=False):
    """main.cu:128-188: sequential-cin accumulation through fp32."""
    r = indices.long()
    acc = x_out[r].clone() if add else torch.zeros((len(r), weight.shape[0]), dtype=x_in.dtype)
    for ci in range(weight.shape[1]):
        acc = acc + x_in[r, ci:ci + 1] * weight[:, ci].view(1, -1)
    if bias is not None:
        acc = acc + bias
    x_out[r] = acc
    return x_out
