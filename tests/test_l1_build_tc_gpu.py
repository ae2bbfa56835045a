"""dagr_l1_build_tc (conv_block1.conv_block1's per-node product on tensor cores, 3xTF32) against dagr_l1_build on the same
inputs: the adjacency (nbr, off, the degree slot) and cellmask are the same bits, xa agrees within 1e-5, and every node's xa
row has the same bits in every instance -- the lean launch with its global-memory fallback (defer = 0) and the regular launch
with the dense kernel behind it (defer = 1).  The adjacency-only form of dagr_l1_build (p_host = NULL) gives the same adjacency
bits.  The stream has a dense cluster so that both fallbacks run."""
import ctypes as C

import pytest
import torch

from tests.helpers import assert_close, make_model

pytestmark = pytest.mark.gpu


def _dense_stream(W, H):
    from dagr_b200.data import EventBatch
    g = torch.Generator().manual_seed(11)
    n_dense, n_bg = 9000, 20000
    x = torch.cat([torch.randint(300, 330, (n_dense,), generator=g), torch.randint(0, W, (n_bg,), generator=g)])
    y = torch.cat([torch.randint(200, 230, (n_dense,), generator=g), torch.randint(0, H, (n_bg,), generator=g)])
    n = n_dense + n_bg
    t = torch.sort(torch.randint(950000, 999999, (n,), generator=g)).values
    perm = torch.randperm(n, generator=g)
    pos_denorm = torch.stack([x[perm], y[perm], t], 1).int()
    p = (torch.randint(0, 2, (n,), generator=g) * 2 - 1).float().view(-1, 1)
    return EventBatch(x=p, pos=torch.zeros(n, 3), batch=torch.zeros(n, dtype=torch.long), width=torch.tensor([W]),
                      height=torch.tensor([H]), time_window=torch.tensor([1000000]), pos_denorm=pos_denorm, num_graphs=1)


def test_tc_build_keeps_the_adjacency_of_both_fp32_forms_and_gives_each_node_the_same_bits_in_every_instance():
    from dagr_b200 import _lib
    W, H = 640, 480
    model, _ = make_model("n", H, W)
    model.cuda()
    eng = model.engine
    batch_i, pos_i, feat, W_, H_ = model._prepare_events(_dense_stream(W, H).cuda())
    eng.forward_events(batch_i, pos_i, feat, 1, W_, H_)
    torch.cuda.synchronize()
    L = eng.last
    geom, ws, N = L["geom"], L["ws"], L["N"]
    lib, pk, g, st, P = eng.lib, eng._pack, C.byref(geom.c_geom), _lib.stream_ptr(), _lib.ptr
    flags = eng._zs(ws, "flags", torch.int32)

    def run(tc, defer, adjacency_only=False):
        nbr, off = torch.zeros_like(ws["nbr"]), torch.zeros_like(ws["off"])
        xa = torch.zeros_like(ws["xa"])
        cellmask = torch.zeros(geom.cells1, dtype=torch.int32, device="cuda")
        wl_hdr = torch.zeros(2, dtype=torch.int32, device="cuda")
        wl_ids = torch.zeros(geom.cells1, dtype=torch.int32, device="cuda")
        head = (g, N, P(ws["start"]), P(ws["ti"]), P(ws["xyb"]), P(ws["feat_s"]))
        tail = (P(flags), 0, P(nbr), P(off), P(cellmask), P(xa), P(wl_hdr), P(wl_ids), defer, st)
        if tc:
            _lib.check(lib.dagr_l1_build_tc(*head, C.byref(pk["l1a"]), P(pk["l1a_wfrag"]), *tail), "l1_build_tc")
        else:
            _lib.check(lib.dagr_l1_build(*head, None if adjacency_only else C.byref(pk["l1a"]), *tail), "l1_build")
        torch.cuda.synchronize()
        return dict(nbr=nbr[:16 * N], off=off[:16 * N], cellmask=cellmask, xa=xa[:2 * N * 8], beyond=int(wl_hdr[0]))

    out = {(tc, defer): run(tc, defer) for tc in (False, True) for defer in (0, 1)}
    for defer in (0, 1):
        plain, tc = out[(False, defer)], out[(True, defer)]
        assert plain["beyond"] > 0 and tc["beyond"] == plain["beyond"], "the stream must exercise the dense fallbacks"
        for k in ("nbr", "off", "cellmask"):
            assert torch.equal(tc[k], plain[k]), (k, defer)
        rows = lambda xa: torch.cat([xa[:N * 8].view(N, 8), xa[N * 8:].view(N, 8)], 1).cpu()
        assert_close(rows(tc["xa"]), rows(plain["xa"]), tol=1e-5, what=f"l1_build_tc vs l1_build xa (defer={defer})")
    assert torch.equal(out[(True, 0)]["xa"], out[(True, 1)]["xa"])
    for defer in (0, 1):
        adj = run(False, defer, adjacency_only=True)
        for k in ("nbr", "off", "cellmask"):
            assert torch.equal(adj[k], out[(False, defer)][k]), ("adjacency only", k, defer)
    # the engine's own forward ran the tensor-core kernel as well
    assert torch.equal(ws["xa"][:2 * N * 8], out[(True, 0)]["xa"]) or torch.equal(ws["xa"][:2 * N * 8], out[(True, 1)]["xa"])
