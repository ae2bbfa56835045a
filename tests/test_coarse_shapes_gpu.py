"""Each coarse kernel of coarse.cu at every shape the shipped configurations launch (tests/shipped_shapes.py derives
them from the models), against the float64 and exact models of tests/test_grid_kernels_cpu.py and
tests/test_grid_kernels_gpu.py, and the derived conv set against the grid_conv labels the engine records.

  * dagr_grid_conv: every derived (Cin, Cout, column block) in every split-K instance it can reach, both tiers (exact
    dyadic inputs with torch.equal, realistic inputs under the float64 bound); the head's prediction convs on both
    halves of their [cells, 2C] input;
  * dagr_grid_linear_bn: every derived (Cin, Cout), with and without the folded BN;
  * dagr_grid_pool / _finalize: every derived pooled width and one that is not a multiple of 32, max and mean, every
    parent field bit for bit;
  * dagr_grid_cat_pos: copy plus position-table lookup, bit for bit, at every derived width;
  * dagr_grid_temporal_filter: pooling.py:69-72 restated on the grid's edge list, bit for bit;
  * dagr_grid_to_dense: the dense maps of the head (cls at ldx nc, reg / obj as column views of ldx 5), with and
    without the CNN maps, bit for bit;
  * dagr_head_finish: nc = 2 and nc = 100, with the CNN maps and with all three NULL.
"""
import numpy as np
import pytest
import torch

from tests.shipped_shapes import config_args, configs, conv_labels, shipped
from tests.test_grid_kernels_cpu import export_grid
from tests.test_grid_kernels_gpu import (CNX, CNY, PH, PW, batch, conv_case, dev, grid, head_finish_case, instance,
                                         linear_bn_case, n_sm, pos_tables, ref_grid_pool, run_grid_pool, sample)

pytestmark = pytest.mark.gpu

SH = shipped()
PER = CNX * CNY


# ------------------------------------------------------------------------------------------------------------------------
# the engine launches exactly the derived convs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size,dataset,use_image", configs(),
                         ids=[f"{s}-{d}-{'image' if i else 'events'}" for s, d, i in configs()])
def test_engine_conv_labels_equal_the_shipped_shapes(size, dataset, use_image):
    """one forward per configuration with per-op timing on: the grid_conv_L{level}_{Cin}x{Cout} labels it records are the
    derived conv set of that configuration"""
    from dagr_b200.data import format_data, synth_batch
    from dagr_b200.model.dagr import DAGR
    W, H, B = 240, 180, 2
    torch.manual_seed(0)
    model = DAGR(config_args(size, dataset, use_image), height=H, width=W).eval().cuda()
    data = format_data(synth_batch(B, 4000, W, H, seed=3, with_image=use_image).clone()).cuda()
    eng = model.engine
    eng.prof = {}
    model.forward_decoded(data)
    torch.cuda.synchronize()
    got = sorted(k for k in eng.prof if k.startswith("grid_conv_"))
    eng.prof = None
    assert got == conv_labels(size, dataset, use_image)


# ------------------------------------------------------------------------------------------------------------------------
# dagr_grid_conv
# ------------------------------------------------------------------------------------------------------------------------
def _conv_cases():
    """(Cin, Cout, off, ldin, size): a dense input at mid and small grids and, where <16> can take it, at a big one; a
    column-block input (the prediction convs) on both halves of its [cells, ldin] array"""
    out = []
    for Cin, Cout, off, ldin in SH["conv"]:
        layouts = [(0, 0)] if ldin == Cin else [(0, ldin), (ldin - Cin, ldin)]
        sizes = (["big"] if instance(Cin, Cout, 10 ** 6, 132) == "sk16" else []) + ["mid", "small"]
        out += [(Cin, Cout, o, ld, s) for o, ld in layouts for s in sizes]
    return out


CONV = _conv_cases()


def test_shipped_conv_cases_reach_every_split_k_instance():
    nsm = n_sm()
    from tests.test_grid_kernels_gpu import NX, NY, batch_for
    got = {instance(ci, co, batch_for(s, nsm) * NX * NY, nsm) for ci, co, _, _, s in CONV}
    assert got == {"sk16", "sk4", "sk1"}, got


@pytest.mark.parametrize("Cin,Cout,off,ldin,size", CONV, ids=[f"{c[0]}x{c[1]}-off{c[2]}-ld{c[3]}-{c[4]}" for c in CONV])
def test_grid_conv_at_shipped_shapes(Cin, Cout, off, ldin, size):
    """the engine's epilogues: folded BN + residual on the layers and the head's hidden convs, bias alone on the
    prediction convs"""
    flags = ("bias",) if ldin else ("bias", "scale", "skip")
    conv_case(Cin, Cout, size, flags=flags, seed=7, off=off, ldin=ldin)


# ------------------------------------------------------------------------------------------------------------------------
# dagr_grid_linear_bn
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", [True, False], ids=["bn", "nobn"])
@pytest.mark.parametrize("Cin,Cout", SH["linear_bn"], ids=[f"{a}x{b}" for a, b in SH["linear_bn"]])
def test_grid_linear_bn_at_shipped_shapes(Cin, Cout, bn):
    linear_bn_case(Cin, Cout, 515, bn)


# ------------------------------------------------------------------------------------------------------------------------
# dagr_grid_pool / _finalize
# ------------------------------------------------------------------------------------------------------------------------
POOL_WIDTHS = sorted({w for w, _ in SH["pool"]} | {50})


@pytest.mark.parametrize("aggr", [0, 1], ids=["max", "mean"])
@pytest.mark.parametrize("C", POOL_WIDTHS)
def test_grid_pool_at_shipped_widths(C, aggr):
    """B = 4 with an empty sample at C channels: the lane loop over channels runs C / 32 passes (and a partial one at 50)"""
    s = batch([sample(1, C), sample(2, C, empty=True), sample(3, C), sample(4, C)])
    got, want = run_grid_pool(s, 4, aggr, C), ref_grid_pool(s, 4, aggr)
    for k in want:
        assert torch.equal(got[k], want[k]), f"C = {C}, {k}: {(got[k] != want[k]).sum()} elements differ"
    assert int(want["pcnt"].gt(1).sum()) > 20


# ------------------------------------------------------------------------------------------------------------------------
# dagr_grid_cat_pos
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cx", SH["cat_pos"])
def test_grid_cat_pos_at_shipped_widths(Cx):
    """xin[cell] = [x[cell], posxr[px], posyr[py]] on valid cells and 0 on empty ones, every element written (NaN
    prefill), B = 3 with an empty sample"""
    from dagr_b200 import _lib
    lib = _lib.load()
    B = 3
    s = batch([sample(11, Cx), sample(12, Cx, empty=True), sample(13, Cx)])
    posxr, posyr = pos_tables()
    cells = B * PER
    cnt, pxy, x = dev(s["cnt"]), dev(s["pxy"]), dev(s["x"])
    xin = torch.full((cells, Cx + 2), float("nan"), device="cuda")
    _lib.check(lib.dagr_grid_cat_pos(grid(CNX, CNY, B, PW, PH, posxr, posyr), _lib.ptr(cnt), _lib.ptr(pxy), _lib.ptr(x), Cx,
                                     _lib.ptr(xin), _lib.stream_ptr()), "dagr_grid_cat_pos")
    torch.cuda.synchronize()
    valid = s["cnt"] > 0
    want = np.zeros((cells, Cx + 2), np.float32)
    want[valid, :Cx] = s["x"][valid]
    want[valid, Cx] = posxr.cpu().numpy()[s["pxy"][valid, 0]]
    want[valid, Cx + 1] = posyr.cpu().numpy()[s["pxy"][valid, 1]]
    assert torch.equal(xin.cpu(), torch.from_numpy(want))
    assert (s["pxy"][valid, 0] != s["pxy"][valid, 1]).mean() > 0.9


# ------------------------------------------------------------------------------------------------------------------------
# dagr_grid_temporal_filter
# ------------------------------------------------------------------------------------------------------------------------
def ref_temporal_filter(cnt, mask, tmax, B):
    """pooling.py:69-72 on the grid: the coarse edges (src -> dst) of the mask keep t_max[dst] > t_max[src]; a valid
    cell's new mask holds the bits of its kept in-edges, an empty cell's mask is left as it was"""
    cells, edges = export_grid(CNX, CNY, B, cnt, mask)
    src, dst = cells[edges[0]].numpy(), cells[edges[1]].numpy()
    keep = tmax[dst] > tmax[src]
    dcx = src % CNX - dst % CNX
    dcy = (src % PER) // CNX - (dst % PER) // CNX
    out = mask.copy()
    out[cnt > 0] = 0
    np.bitwise_or.at(out, dst[keep], (1 << ((dcy + 1) * 3 + dcx + 1))[keep].astype(out.dtype))
    return out, tmax[dst] == tmax[src]


def test_grid_temporal_filter_vs_the_edge_list_model():
    """B = 4 with an empty sample; t_max drawn from 9 levels (ties: the strict > matters); mask bits pointing at empty
    cells, off the grid, across the sample boundary and at the centre"""
    from dagr_b200 import _lib
    lib = _lib.load()
    B = 4
    s = batch([sample(21), sample(22, empty=True), sample(23), sample(24)])
    d_cnt, d_tmax, d_mask = dev(s["cnt"]), dev(s["tmax"]), dev(s["mask"].copy())
    _lib.check(lib.dagr_grid_temporal_filter(grid(CNX, CNY, B), _lib.ptr(d_cnt), _lib.ptr(d_tmax), _lib.ptr(d_mask),
                                             _lib.stream_ptr()), "dagr_grid_temporal_filter")
    torch.cuda.synchronize()
    want, tie = ref_temporal_filter(s["cnt"], s["mask"], s["tmax"], B)
    got = d_mask.cpu().numpy()
    assert np.array_equal(got, want), f"{(got != want).sum()} cells differ"
    # the input really has every edge case
    valid = s["cnt"] > 0
    cy = (np.arange(B * PER) % PER) // CNX
    assert tie.sum() > 10
    assert (valid & ((s["mask"] >> 4) & 1).astype(bool)).sum() > 10                                    # centre bit
    assert (valid & (cy == CNY - 1) & ((s["mask"] >> 7) & 1).astype(bool)).sum() > 3                  # across samples
    assert (valid & ~np.roll(valid, -1) & ((s["mask"] >> 5) & 1).astype(bool)).sum() > 10              # empty neighbour
    assert (~valid & (s["mask"] != 0)).sum() > 10                                                      # untouched


# ------------------------------------------------------------------------------------------------------------------------
# dagr_grid_to_dense
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,ldx,off,with_add", SH["to_dense"] + [(16, 0, 0, True)],
                         ids=[f"C{c}-ld{l}-off{o}-{'add' if a else 'noadd'}" for c, l, o, a in SH["to_dense"] + [(16, 0, 0, True)]])
def test_grid_to_dense_at_shipped_views(C, ldx, off, with_add):
    """dense[b, c, y, x] = (valid ? x[cell, off + c] : 0) + add[b, c, y, x]: columns [off, off + C) of a [cells, ldx]
    array (ldx = 0: a dense [cells, C] one), B = 3 with an empty sample, NaN prefill"""
    from dagr_b200 import _lib
    lib = _lib.load()
    B = 3
    rng = np.random.default_rng([C, ldx, off, with_add])
    s = batch([sample(31), sample(32, empty=True), sample(33)])
    cells = B * PER
    width = ldx or C
    x = rng.standard_normal((cells, width)).astype(np.float32)
    add = rng.standard_normal((B, C, CNY, CNX)).astype(np.float32) if with_add else None
    d_cnt, d_x = dev(s["cnt"]), dev(x)
    d_add = dev(add) if with_add else None
    dense = torch.full((B, C, CNY, CNX), float("nan"), device="cuda")
    _lib.check(lib.dagr_grid_to_dense(grid(CNX, CNY, B), _lib.ptr(d_cnt), _lib.ptr(d_x[:, off:]), C, ldx,
                                      _lib.ptr(d_add), _lib.ptr(dense), _lib.stream_ptr()), "dagr_grid_to_dense")
    torch.cuda.synchronize()
    v = np.where((s["cnt"] > 0)[:, None], x[:, off:off + C], np.float32(0))
    want = v.reshape(B, CNY, CNX, C).transpose(0, 3, 1, 2)
    if with_add:
        want = want + add
    assert torch.equal(dense.cpu(), torch.from_numpy(np.ascontiguousarray(want, np.float32)))


# ------------------------------------------------------------------------------------------------------------------------
# dagr_head_finish
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("maps", [True, False], ids=["cnn_maps", "events_only"])
@pytest.mark.parametrize("nc", sorted({nc for nc, _ in SH["head_finish"]}))
def test_head_finish_at_shipped_class_counts(nc, maps):
    """nc = 2 (DSEC) and 100 (N-Caltech101); the events-only models pass NULL for all three CNN maps"""
    assert (nc, maps) in SH["head_finish"]
    head_finish_case(nc, maps)
