"""The radius graph at its decision edges, on the device: the hand-placed cases of tests/test_radius_graph_edges_cpu.py.

Each case runs dagr_graph_sort, then dagr_l1_build (adjacency only) with flags = NULL and with the sort's flags, then
dagr_graph_export: the edge_index must equal the graph oracle's bit for bit.  dagr_l1_build_tc with the sort's flags, at
defer 0 and 1, must give the same adjacency (nbr, off, degree slot 15, cellmask) as test_l1_kernels_gpu.Stream derives from the
oracle.  An incremental case (min_idx > 0) compares the rows of the new nodes.  Then the time-order defects through the model:
interleaved samples at B = 2 must give the oracle's edges from model(data), and a bench-shaped batch (contiguous, time-sorted
samples) must leave the sort's flag clear, so the product keeps its time-bucket pruning.
"""
import numpy as np
import pytest
import torch

from tests.test_l1_kernels_gpu import P, Stream, _lib, build_params, l1a, new_mask, run_build, st
from tests.test_radius_graph_edges_cpu import CASES, build_case, regimes

pytestmark = pytest.mark.gpu


def export(s, nbr):
    """dagr_graph_export of an ELL [16, N] (sorted positions) -> edge_index int64 [2, E] (arrival ids)"""
    L, lib = _lib()
    N = s.N
    d_nbr = nbr.int().reshape(-1).cuda()
    inv = torch.zeros(N, dtype=torch.int32, device="cuda")
    rowptr = torch.zeros(N + 1, dtype=torch.int32, device="cuda")
    blocksums = torch.zeros(int(lib.dagr_scan_blocks(N + 1)) + 2, dtype=torch.int32, device="cuda")
    es = torch.zeros(16 * N, dtype=torch.int64, device="cuda")
    ed = torch.zeros(16 * N, dtype=torch.int64, device="cuda")
    L.check(lib.dagr_graph_export(None, N, P(s.perm_d), P(s.ti), P(d_nbr), P(inv), P(rowptr), P(blocksums), P(es), P(ed), 16 * N,
                                  st()), "export")
    torch.cuda.synchronize()
    E = int(rowptr[N])
    return torch.stack([es[:E], ed[:E]]).cpu()


def case_stream(name):
    c = build_case(name)
    g = c.geo
    flag = regimes(c.geometry(), c.batch.numpy(), c.pos.numpy(), c.min_idx)["flag"]
    s = Stream(g["W"], g["H"], g["B"], 0, 0, radius=g["radius"], K=g["K"], events=(c.batch, c.pos), time_window=g["T"],
               max_queue_size=g["Q"], expect_flag=int(flag))
    return c, s


def same_rows(o, want, rows, what):
    nbr, off, deg = want
    valid = (nbr >= 0) & rows[None, :]
    assert torch.equal(o["nbr"][valid], nbr[valid]) and torch.equal(o["off"][valid], off[valid]), what
    assert torch.equal(o["nbr"][15][rows], deg[rows]), what


@pytest.mark.parametrize("name", list(CASES))
def test_case_edges_equal_the_oracle(name):
    c, s = case_stream(name)
    nbr, off, deg, mask, _ = s.expected_adjacency()
    m = c.min_idx
    rows = s.perm >= m                                              # sorted positions of the nodes this launch processes
    for flags in (None, s.flags):
        what = (name, "flags" if flags is not None else "NULL")
        a = run_build(s, None, None, 1, tc=False, flags=flags, min_idx=m)
        if m == 0:
            got = export(s, a["nbr"])
            assert torch.equal(got, s.edges), (what, got.shape, s.edges.shape)
        same_rows(a, (nbr, off, deg), rows, what)
    pa, wf = l1a(build_params(np.random.default_rng(0), False))
    for defer in (0, 1):
        o = run_build(s, pa, wf, defer, flags=s.flags, min_idx=m)
        same_rows(o, (nbr, off, deg), rows, (name, "tc", defer))
        assert torch.equal(o["cellmask"], mask if m == 0 else new_mask(s, m)), (name, "tc", defer)


def sort_flag(model):
    eng = model.engine
    return int(eng._zs(eng.last["ws"], "flags", torch.int32)[0])


def _model_edges(W, H, B, batch, pos):
    from dagr_b200.data import EventBatch
    from tests.helpers import make_model
    from oracle import ref_ops as R
    model, args = make_model("n", H, W)
    model.cuda()
    n = len(batch)
    data = EventBatch(x=torch.ones(n, 1), pos=torch.zeros(n, 3), batch=batch.long(), width=torch.tensor([W]),
                      height=torch.tensor([H]), time_window=torch.tensor([1000000]), pos_denorm=pos.int(), num_graphs=B)
    model(data.clone().cuda())
    torch.cuda.synchronize()
    g = R.RefGraph(W, H, B, args.max_neighbors, 128, int(args.radius * W + 1), int(args.radius * 1000000))
    return model, model.engine.export_edges().cpu(), g.forward(batch.int(), pos.int())


def test_model_keeps_the_edge_of_an_inversion_between_interleaved_samples():
    """B = 2 with sample ids 0, 1, 0: arrival 2 at (101, 100), t = 960000 reads arrival 0 at (100, 100), t = 990000 (dt < 0).
    Then time-sorted background: sample 1 anywhere, then sample 0 away from that pixel's voxel (which keeps spanning 4 slices)"""
    W, H = 240, 180
    rng = np.random.default_rng(3)
    n = 2000
    b = np.repeat([1, 0], n)
    t = np.concatenate([np.sort(rng.integers(970000, 1000000, n)), np.sort(rng.integers(900000, 1000000, n))])
    x = np.concatenate([rng.integers(0, W, n), rng.integers(0, 60, n)])
    y = rng.integers(0, H, 2 * n)
    pre = np.array([[0, 100, 100, 990000], [1, 50, 50, 970000], [0, 101, 100, 960000]])
    ev = np.concatenate([pre, np.stack([b, x, y, t], 1)])
    batch, pos = torch.from_numpy(ev[:, 0]), torch.from_numpy(ev[:, 1:])
    model, got, want = _model_edges(W, H, 2, batch, pos)
    assert ((want[0] == 0) & (want[1] == 2)).any(), "the oracle has the edge 0 -> 2"
    assert torch.equal(got, want)
    assert sort_flag(model) == 1


def test_bench_shaped_batch_keeps_the_flag_clear():
    """B = 8 contiguous samples of 50 ms windows (data.synth_batch, as bench.py): the sort proves the time order, so the build
    prunes by time"""
    from dagr_b200.data import format_data, synth_batch
    from tests.helpers import make_model
    W, H = 640, 480
    model, _ = make_model("n", H, W)
    model.cuda()
    data = format_data(synth_batch(8, 20000, W, H, seed=4242))
    model(data.clone().cuda())
    torch.cuda.synchronize()
    assert model.engine.last["N"] == 8 * 20000
    assert sort_flag(model) == 0
