"""Host-side geometry of one (width, height, batch, radius) configuration.

Every table is built with the SAME fp32 torch ops the reference executes so that integer
results derived from floating point (voxel ids, rounded pixel positions, dense-grid indices)
are bit-exact (SURVEY H2): never a reciprocal multiply where the reference divides.

reference formulas:
  pos = int / int  true division            src/dagr/utils/buffers.py:33-44
  voxel sizes (1/7,1/5)/2^(3-i)             src/dagr/model/networks/net.py:19-28
  grid_cluster trunc(pos/size)              src/dagr/model/layers/pooling.py:55-56 (torch_cluster)
  round_to_pixel                            pooling.py:47-49
  spiral probe order                        src/dagr/graph/spiral.h:1-16
  LUT basis at integer offsets              src/dagr/model/layers/spline_conv.py:16-37
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import List, Tuple

import numpy as np
import torch

from . import _lib


def spiral_offsets(r: int) -> torch.Tensor:
    """first (2r+1)^2 cells of SpiralOut (spiral.h): int8 [ncell, 2] = (dx, dy)."""
    n = (2 * r + 1) ** 2
    out = np.zeros((n, 2), dtype=np.int8)
    layer, leg, x, y = 1, 0, 0, 0
    for i in range(n):
        out[i] = (x, y)
        if leg == 0:
            x += 1
            if x == layer:
                leg += 1
        elif leg == 1:
            y += 1
            if y == layer:
                leg += 1
        elif leg == 2:
            x -= 1
            if -x == layer:
                leg += 1
        else:
            y -= 1
            if -y == layer:
                leg = 0
                layer += 1
    return torch.from_numpy(out)


def compute_pooling_at_each_layer(pooling_dim_at_output: str, num_layers: int = 4) -> torch.Tensor:
    """net.py:19-28."""
    py, px = map(int, str(pooling_dim_at_output).split("x"))
    base = torch.tensor([1.0 / px, 1.0 / py, 1.0 / 1])
    out = []
    for i in range(num_layers):
        p = base / 2 ** (3 - i)
        p[-1] = 1
        out.append(p)
    return torch.stack(out)


def spline_basis_deg1(pseudo: torch.Tensor, ks: int = 5):
    """degree-1 open B-spline basis (published torch_spline_conv algorithm): basis[E,4], slot[E,4]."""
    E, dim = pseudo.shape
    S = 2 ** dim
    basis = torch.ones((E, S), dtype=pseudo.dtype)
    index = torch.zeros((E, S), dtype=torch.long)
    mult = 1
    for d in range(dim):
        v = pseudo[:, d] * float(ks - 1)
        frac = v - torch.floor(v)
        for s in range(S):
            k = (s >> d) & 1
            index[:, s] += ((v.to(torch.long) + k) % ks) * mult
            basis[:, s] = basis[:, s] * (frac if k == 1 else (1 - frac))
        mult *= ks
    return basis, index


@dataclass
class Level:
    """one pooled voxel grid (pool1..pool4)."""
    nx: int
    ny: int
    voxel: torch.Tensor            # fp32 [3] voxel size (pooling.py:24)
    cart_max: object               # max_value of the T.Cartesian transform after this pooling (net.py:77-95)
    cellx: torch.Tensor            # int32 [W] pixel (rounded pos) -> voxel x index
    celly: torch.Tensor            # int32 [H]
    den_x: float                   # fl32(2*M*W) used by init_lut for convs AFTER this pooling
    den_y: float
    grid: _lib.Grid = None
    cellx_dev: torch.Tensor = None
    celly_dev: torch.Tensor = None


class Geometry:
    def __init__(self, width: int, height: int, batch_size: int, radius: float = 0.01, time_window: int = 1000000,
                 max_neighbors: int = 16, max_queue_size: int = 128, pooling_dim_at_output: str = "5x7",
                 kernel_size: int = 5, device="cuda"):
        W, H, B = int(width), int(height), int(batch_size)
        self.W, self.H, self.B, self.T = W, H, B, int(time_window)
        self.radius = radius
        self.r = int(radius * W + 1)                         # ev_tgn.py:29
        self.dt_us = int(radius * time_window)               # ev_tgn.py:28
        self.K, self.Q = int(max_neighbors), int(max_queue_size)
        self.ncell = (2 * self.r + 1) ** 2
        self.kernel_size = kernel_size
        if self.K < 1 or self.K > _lib.ELL:
            raise ValueError("max_neighbors must be in [1, 16]")
        if kernel_size != 5:
            raise ValueError("only kernel_size 5 (the reference configs) is supported")

        # ---- normalised positions -----------------------------------------------------------
        self.posx0 = torch.arange(W, dtype=torch.int32) / torch.tensor(W)        # buffers.py:43
        self.posy0 = torch.arange(H, dtype=torch.int32) / torch.tensor(H)
        wh_inv = 1 / torch.Tensor([[W, H]])                                      # pooling.py:32
        self.posxr = torch.arange(W).float() * wh_inv[0, 0]                      # round_to_pixel product
        self.posyr = torch.arange(H).float() * wh_inv[0, 1]

        # ---- voxel grids ----------------------------------------------------------------------
        poolings = compute_pooling_at_each_layer(pooling_dim_at_output, 4)
        self.poolings = poolings
        max_vals = 2 * poolings[:, :2].max(-1).values                            # net.py:68
        self.effective_radius = 2 * float(int(radius * W + 2) / W)               # net.py:72
        cart_max = [2 * self.effective_radius, max_vals[1], max_vals[2], max_vals[3]]
        end = torch.tensor(0.9999999)
        self.levels: List[Level] = []
        for i in range(4):
            size = poolings[i]
            src_x = self.posx0 if i == 0 else self.posxr
            src_y = self.posy0 if i == 0 else self.posyr
            cellx = (src_x / size[0]).to(torch.long)                             # grid_cluster (fp32 division)
            celly = (src_y / size[1]).to(torch.long)
            nx = int(((end - 0) / size[0]).to(torch.long)) + 1
            ny = int(((end - 0) / size[1]).to(torch.long)) + 1
            if int(cellx.max()) >= nx or int(celly.max()) >= ny:
                raise ValueError("voxel index exceeds the grid computed by grid_cluster")
            M = cart_max[i]
            den_x = float(torch.tensor(2 * M * W, dtype=torch.float32)) if not torch.is_tensor(M) else float(2 * M * W)
            den_y = float(torch.tensor(2 * M * H, dtype=torch.float32)) if not torch.is_tensor(M) else float(2 * M * H)
            self.levels.append(Level(nx=nx, ny=ny, voxel=size.clone(), cart_max=M, cellx=cellx.int(), celly=celly.int(),
                                     den_x=den_x, den_y=den_y))

        # ---- cell-major sort key (level-1 voxels) --------------------------------------------
        l1 = self.levels[0]
        self.nx1, self.ny1 = l1.nx, l1.ny
        cx, cy = l1.cellx.long(), l1.celly.long()
        if not (torch.all(cx[1:] >= cx[:-1]) and torch.all(cy[1:] >= cy[:-1])):
            raise ValueError("voxel LUT is not monotone")
        x0 = torch.full((self.nx1,), W, dtype=torch.long).scatter_reduce(0, cx, torch.arange(W), reduce="amin")
        y0 = torch.full((self.ny1,), H, dtype=torch.long).scatter_reduce(0, cy, torch.arange(H), reduce="amin")
        self.CW = int(torch.bincount(cx, minlength=self.nx1).max())
        self.CH = int(torch.bincount(cy, minlength=self.ny1).max())
        self.CP = self.CW * self.CH
        minw = int(torch.bincount(cx, minlength=self.nx1)[: int(cx.max()) + 1].min())
        minh = int(torch.bincount(cy, minlength=self.ny1)[: int(cy.max()) + 1].min())
        if self.r >= min(minw, minh):
            raise ValueError(f"event radius {self.r}px must be smaller than a pool1 voxel ({minw}x{minh}px): "
                             "coarse edges would span more than the 8-neighbourhood")
        self.vx0 = torch.cat([x0, torch.tensor([W])]).int()
        self.vy0 = torch.cat([y0, torch.tensor([H])]).int()
        if int(cx.max()) + 1 != self.nx1 or int(cy.max()) + 1 != self.ny1:
            raise ValueError("empty voxel columns/rows in the pool1 grid")
        self.xkey = (cx * self.CP + (torch.arange(W) - x0[cx])).int()
        self.ykey = (cy * self.nx1 * self.CP + (torch.arange(H) - y0[cy]) * self.CW).int()
        self.NK = B * self.ny1 * self.nx1 * self.CP
        if self.NK >= 1 << 31:
            raise ValueError(f"{B} x {self.ny1} x {self.nx1} pool1 voxels of {self.CP} pixels give {self.NK} sort keys: the "
                             "graph sort's 32-bit sort key holds fewer than 2^31")
        self.cells1 = B * self.ny1 * self.nx1
        self.spiral = spiral_offsets(self.r)

        # ---- event-level offset table (init_lut at integer offsets, spline_conv.py:16-37) -----
        M = self.effective_radius                                 # dagr.py:38
        d = self.spiral.float()
        ax = d[:, 0] / (2 * M * W) + 0.5
        ay = d[:, 1] / (2 * M * H) + 0.5
        basis, slot = spline_basis_deg1(torch.stack([ax, ay], dim=1), kernel_size)
        # reachable spline kernels form a product grid xs x ys (<= 3 x 5): slot id = sx + ks*sy
        nz = slot[basis != 0]
        xs = sorted(set((nz % kernel_size).tolist()) | {int(slot[0, 0]) % kernel_size})
        ys = sorted(set((nz // kernel_size).tolist()) | {int(slot[0, 0]) // kernel_size})
        if len(xs) > 3 or len(ys) > 5:
            raise ValueError("more than 3 x 5 spline kernel slots reachable at the event level")
        xs = xs + [u for u in range(kernel_size) if u not in xs][: 3 - len(xs)]
        ys = ys + [u for u in range(kernel_size) if u not in ys][: 5 - len(ys)]
        self.slots_x, self.slots_y = xs, ys
        used = [xs[i] + kernel_size * ys[j] for j in range(5) for i in range(3)]
        self.den1_x = float(torch.tensor(2 * M * W, dtype=torch.float32))      # init_lut divisor (spline_conv.py:28-29)
        self.den1_y = float(torch.tensor(2 * M * H, dtype=torch.float32))
        self.slots1 = used                                         # slot ids, length 15 = 5 (y) x 3 (x)
        tab = torch.zeros((self.ncell, _lib.TABW), dtype=torch.float32)
        for s in range(4):
            for u, sl in enumerate(used):
                m = slot[:, s] == sl
                tab[m, u] += basis[m, s]
        self.tab1 = tab
        # the table is a product: tab[c][k + 3 j] = tabx[dx + r][k] * taby[dy + r][j] (one bilinear factor per axis);
        # conv_b rebuilds the 15 weights from the two factors (8 floats instead of 16 per edge)
        cell_of = {(int(dx), int(dy)): c for c, (dx, dy) in enumerate(self.spiral.tolist())}
        c0 = tab[0, :15].reshape(5, 3)
        j0, k0 = [int(v) for v in torch.nonzero(c0 == 1.0)[0]]
        r = self.r
        tabx = torch.zeros((2 * r + 1, 4), dtype=torch.float32)
        taby = torch.zeros((2 * r + 1, 8), dtype=torch.float32)
        for i in range(-r, r + 1):
            tabx[i + r, :3] = tab[cell_of[(i, 0)], :15].reshape(5, 3)[j0]
            taby[i + r, :5] = tab[cell_of[(0, i)], :15].reshape(5, 3)[:, k0]
        dxs, dys = self.spiral[:, 0].long() + r, self.spiral[:, 1].long() + r
        prod = (taby[dys, :5].unsqueeze(2) * tabx[dxs, :3].unsqueeze(1)).reshape(-1, 15)
        if not torch.equal(prod, tab[:, :15]):
            raise ValueError("event-level slot table is not an exact product of per-axis factors")
        self.tabx, self.taby = tabx, taby

        # den for event-level LUT: same expression as init_lut
        self.device = torch.device(device)
        self._upload()

    # ------------------------------------------------------------------------------------------
    def _upload(self):
        dev = self.device
        self.d_xkey = self.xkey.to(dev)
        self.d_ykey = self.ykey.to(dev)
        self.d_spiral = self.spiral.to(dev)
        self.d_posx0 = self.posx0.to(dev)
        self.d_posy0 = self.posy0.to(dev)
        self.d_posxr = self.posxr.to(dev)
        self.d_posyr = self.posyr.to(dev)
        self.d_tabx = self.tabx.to(dev)
        self.d_taby = self.taby.to(dev)
        self.d_vx0 = self.vx0.to(dev)
        self.d_vy0 = self.vy0.to(dev)
        g = _lib.Geom()
        g.W, g.H, g.B, g.T = self.W, self.H, self.B, self.T
        g.r, g.ncell = self.r, self.ncell
        g.dt_us, g.K, g.Q = self.dt_us, self.K, self.Q
        g.nx1, g.ny1 = self.nx1, self.ny1
        g.CW, g.CH, g.CP = self.CW, self.CH, self.CP
        g.NK = self.NK
        g.xkey = self.d_xkey.data_ptr(); g.ykey = self.d_ykey.data_ptr()
        g.spiral = self.d_spiral.data_ptr()
        g.posx0 = self.d_posx0.data_ptr(); g.posy0 = self.d_posy0.data_ptr()
        g.vx0 = self.d_vx0.data_ptr(); g.vy0 = self.d_vy0.data_ptr()
        g.tabx = self.d_tabx.data_ptr(); g.taby = self.d_taby.data_ptr()
        self.c_geom = g
        for lv in self.levels:
            gr = _lib.Grid()
            gr.nx, gr.ny, gr.B, gr.W, gr.H = lv.nx, lv.ny, self.B, self.W, self.H
            gr.posxr = self.d_posxr.data_ptr(); gr.posyr = self.d_posyr.data_ptr()
            lv.grid = gr
            lv.cellx_dev = lv.cellx.to(dev)
            lv.celly_dev = lv.celly.to(dev)

    def cells(self, level: int) -> int:
        lv = self.levels[level]
        return self.B * lv.nx * lv.ny
