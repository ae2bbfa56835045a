"""CPU suite: the oracle against its fixed points, host logic, and the C-ABI surface (no GPU)."""
import ctypes
import json
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import ref_ops as R
from tests.helpers import assert_close, make_inputs, make_model

ROOT = Path(__file__).resolve().parent.parent
GOLD = ROOT / "tests" / "golden"


# ---------------------------------------------------------------------------------------------
# spline basis KATs (SURVEY 8c)
# ---------------------------------------------------------------------------------------------
def test_spline_basis_kats_oracle_and_product_tables():
    from dagr_b200.geometry import spline_basis_deg1
    k = json.loads((GOLD / "spline_kats.json").read_text())
    for fn in (lambda p: R.spline_basis(p, 5, True, 1), lambda p: spline_basis_deg1(p, 5)):
        p1 = torch.tensor(k["one_d"]["pseudo"]).view(-1, 1)
        b, i = fn(p1)
        assert torch.allclose(b, torch.tensor(k["one_d"]["basis"], dtype=torch.float32))
        assert i.tolist() == k["one_d"]["index"]
        p2 = torch.tensor(k["two_d"]["pseudo"])
        b, i = fn(p2)
        assert torch.allclose(b, torch.tensor(k["two_d"]["basis"], dtype=torch.float32))
        assert i.tolist() == k["two_d"]["index"]
        r = torch.rand(1000, 2)
        b, _ = fn(r)
        assert torch.allclose(b.sum(1), torch.ones(1000), atol=1e-6)      # partition of unity


def test_lut_equals_basis_form():
    torch.manual_seed(0)
    W, H = 640, 480
    w = torch.randn(25, 5, 7)
    rx, ry, M = R.lut_params_layer1(0.01, W)
    lut, remap = R.build_lut(w, H, W, rx, M)
    # integer offsets -> attrs exactly as Cartesian would produce them up to fp32 noise
    d = torch.stack(torch.meshgrid(torch.arange(-rx, rx + 1), torch.arange(-ry, ry + 1), indexing="ij")).view(2, -1).t().float()
    attr = torch.stack([d[:, 0] / W / (2 * M) + 0.5, d[:, 1] / H / (2 * M) + 0.5], 1)
    x = torch.randn(len(d), 5)
    m_lut = R.message_lut(x, attr, lut, remap)
    b, i = R.spline_basis(attr, 5, True, 1)
    m_bas = R.spline_weighting(x, w, b, i)
    assert_close(m_lut, m_bas, tol=1e-4, what="LUT vs basis form")


# ---------------------------------------------------------------------------------------------
# graph oracle: hand-checkable cases restating ev_graph.cu semantics
# ---------------------------------------------------------------------------------------------
def test_spiral_order_matches_spiral_h():
    from dagr_b200.geometry import spiral_offsets
    s = spiral_offsets(2).tolist()
    assert s[:18] == [[0, 0], [1, 0], [1, 1], [0, 1], [-1, 1], [-1, 0], [-1, -1], [0, -1], [1, -1], [2, -1], [2, 0],
                      [2, 1], [2, 2], [1, 2], [0, 2], [-1, 2], [-2, 2], [-2, 1]]
    for r in (3, 4, 7):
        s = spiral_offsets(r)
        assert len(set(map(tuple, s.tolist()))) == (2 * r + 1) ** 2
        assert int(s.abs().max()) == r


def _edges(g, batch, pos):
    return g.forward(torch.tensor(batch, dtype=torch.int32), torch.tensor(pos, dtype=torch.int32))


def test_graph_oracle_basic_semantics():
    g = R.RefGraph(16, 16, batch_size=2, max_num_neighbors=4, max_queue_size=3, radius=2, delta_t_us=100)
    # events: (x,y,t); same pixel history, dt filter, causality, K cap, batches separated
    batch = [0, 0, 0, 0, 1, 1]
    pos = [[5, 5, 0], [5, 5, 50], [6, 5, 120], [5, 5, 130], [5, 5, 10], [5, 6, 20]]
    e = _edges(g, batch, pos)
    got = list(zip(e[0].tolist(), e[1].tolist()))
    # node 0: self. node 1: self, 0 (dt 50). node 2 (t=120): self, then spiral cell (-1,0)=px(5,5): newest first
    #   idx3 is newer (skipped), idx1 dt=70 ok, idx0 dt=120 > 100 skipped.
    # node 3 (t=130): self; own pixel: idx1 dt 80 ok, idx0 dt 130 no; then (1,0)=px(6,5): idx2 dt 10 ok
    # node 4 (batch 1): self.  node 5: self, then (0,-1)... spiral reaches (0,-1) = px(5,5) of batch 1: idx4
    assert got == [(0, 0), (1, 1), (0, 1), (2, 2), (1, 2), (3, 3), (1, 3), (2, 3), (4, 4), (5, 5), (4, 5)]
    # K cap = 4 incl. self loop; FIFO depth 3 keeps only the newest 3 per pixel
    g = R.RefGraph(8, 8, 1, max_num_neighbors=4, max_queue_size=3, radius=1, delta_t_us=1000)
    e = _edges(g, [0] * 6, [[3, 3, i] for i in range(6)])
    dst5 = e[0][e[1] == 5].tolist()
    assert dst5 == [5, 4, 3]          # self, then FIFO = [5,4,3] (newest 3): 5 is not < own; 4, 3 accepted
    dst2 = e[0][e[1] == 2].tolist()
    assert dst2 == [2]                # FIFO of the pixel holds [5,4,3] only: nothing older than 2 is visible


def test_graph_oracle_single_event_goes_to_batch0_and_empty_input():
    g = R.RefGraph(8, 8, 2, 16, 8, 1, 1000)
    assert g.forward(torch.zeros(0, dtype=torch.int32), torch.zeros((0, 3), dtype=torch.int32)).shape == (2, 0)
    e = _edges(g, [1], [[2, 2, 5]])               # single-event kernel ignores batch (ev_graph.cu:150-152)
    assert e.tolist() == [[0], [0]]
    e = _edges(g, [0, 0], [[2, 2, 6], [3, 2, 7]])  # no reset: indices continue, node 0 is visible in batch 0
    assert list(zip(e[0].tolist(), e[1].tolist())) == [(1, 1), (0, 1), (2, 2), (1, 2), (0, 2)]


def test_denormalize_roundtrip_exact():
    W, H, T = 640, 480, 1000000
    xy = torch.stack([torch.arange(W).repeat_interleave(3)[:1440] % W, torch.arange(1440) % H], 1).to(torch.int16)
    t = torch.randint(0, T, (1440,), dtype=torch.int32)
    pos = R.format_pos(xy, t, W, H, T)
    back = R.denormalize_pos(pos, W, H, T)
    assert torch.equal(back[:, :2], xy.int())           # pixel coordinates survive the fp32 round trip
    # timestamps do NOT always survive it ((t/T)*T + 1e-3 truncates to t-1 for some t > 2^17): that is the
    # reference's own behaviour (ev_tgn.py:15-16) and the product mirrors the same fp32 ops bit for bit
    assert int((back[:, 2] - t).abs().max()) <= 1 and bool((back[:, 2] <= t).all())


# ---------------------------------------------------------------------------------------------
# geometry: fp32-exact voxel LUTs reproduce grid_cluster
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H", [(640, 480), (320, 215), (240, 180)])
def test_geometry_voxel_luts_match_grid_cluster(W, H):
    from dagr_b200.geometry import Geometry
    B = 3
    geom = Geometry(W, H, B, device="cpu")
    poolings = R.compute_pooling_at_each_layer("5x7", 4)
    xs = torch.arange(W).repeat(H)
    ys = torch.arange(H).repeat_interleave(W)
    for lv in range(4):
        if lv == 0:
            pos = torch.stack([xs.int() / torch.tensor(W), ys.int() / torch.tensor(H), torch.zeros(len(xs))], 1)
        else:
            wh_inv = 1 / torch.Tensor([[W, H]])
            pos = torch.cat([torch.stack([xs, ys], 1).float() * wh_inv, torch.zeros(len(xs), 1)], 1)
        for b in (0, B - 1):
            pos4 = torch.cat([pos, torch.full((len(xs), 1), float(b))], 1)
            size = torch.cat([poolings[lv], torch.Tensor([1])])
            c = R.grid_cluster(pos4, size, torch.zeros(4), torch.Tensor([0.9999999, 0.9999999, 0.9999999, B - 1]))
            L = geom.levels[lv]
            mine = L.cellx[xs].long() + L.nx * L.celly[ys].long() + L.nx * L.ny * b
            assert torch.equal(c, mine), f"level {lv} batch {b}"
    # the fp32 quirk columns found by the survey (H2)
    if (W, H) == (640, 480):
        exact = torch.arange(W) * 56 // W
        assert torch.nonzero(geom.levels[0].cellx.long() != exact).flatten().tolist() == [80, 160, 320, 560]
    # sort key is a bijection pixel -> (voxel, slot)
    key = geom.ykey[ys].long() + geom.xkey[xs].long()
    assert len(torch.unique(key)) == W * H
    assert torch.equal(key // geom.CP, geom.levels[0].cellx[xs].long() + geom.nx1 * geom.levels[0].celly[ys].long())


def test_event_level_table_reproduces_lut():
    from dagr_b200.geometry import Geometry
    torch.manual_seed(1)
    W, H = 640, 480
    geom = Geometry(W, H, 1, device="cpu")
    w = torch.randn(25, 3, 4)
    rx, ry, M = R.lut_params_layer1(0.01, W)
    lut, _ = R.build_lut(w, H, W, rx, M)
    slots = torch.tensor(geom.slots1)
    for c in (0, 1, 17, 100, 224):
        dx, dy = geom.spiral[c].tolist()
        mine = (geom.tab1[c, :15].view(-1, 1, 1) * w[slots]).sum(0)
        assert torch.allclose(mine, lut[dx + rx, dy + ry], atol=1e-6)


# ---------------------------------------------------------------------------------------------
# pooling / nms / masked ops of the oracle: small known answers
# ---------------------------------------------------------------------------------------------
def test_oracle_pooling_small_known_answer():
    W, H, B = 640, 480, 1
    poolings = R.compute_pooling_at_each_layer("5x7", 4)
    # 3 events: two in voxel (0,0), one in voxel (1,0); edge 0->1 (same voxel, dropped), 0->2 and 1->2 (dedup)
    xy = torch.tensor([[1, 1], [4, 3], [13, 2]], dtype=torch.int16)
    pos = R.format_pos(xy, torch.tensor([10, 20, 30], dtype=torch.int32), W, H, 1000000)
    x = torch.tensor([[1.0, -1.0], [0.5, 2.0], [3.0, 0.0]])
    ei = torch.tensor([[0, 0, 1, 1, 0, 2, 1], [0, 1, 1, 2, 2, 2, 2]])
    out = R.pooling(x, pos, torch.zeros(3, dtype=torch.long), ei, poolings[0], W, H, B, 0.05)
    assert out["x"].tolist() == [[1.0, 2.0], [3.0, 0.0]]
    assert out["edge_index"].tolist() == [[0], [1]]
    px = (out["pos"][:, :2] * torch.tensor([W, H])).round().long().tolist()
    assert px == [[2, 2], [13, 2]]                       # mean (2.5,2) floored to pixel; single event unchanged


def test_oracle_nms_and_postprocess_quirk():
    boxes = torch.tensor([[0, 0, 10, 10], [1, 1, 11, 11], [20, 20, 30, 30]], dtype=torch.float32)
    keep = R.nms(boxes, torch.tensor([0.9, 0.8, 0.7]), 0.5)
    assert keep.tolist() == [0, 2]
    # confidence filter uses obj*cls^2 (model/utils.py:80-82)
    pred = torch.tensor([[[5., 5., 10., 10., 0.1, 0.09, 0.02], [50., 50., 10., 10., 0.5, 0.5, 0.1]]])
    det = R.postprocess_network_output(pred, 2, conf_thre=0.001, nms_thre=0.65)[0]
    assert len(det["boxes"]) == 1 and abs(float(det["scores"][0]) - 0.25) < 1e-7


def test_oracle_masked_ops():
    torch.manual_seed(0)
    x = torch.randn(10, 4); w = torch.randn(3, 4); b = torch.randn(3)
    out = torch.zeros(10, 3)
    R.masked_lin(torch.tensor([1, 7]), x, out, w, b)
    assert torch.allclose(out[[1, 7]], x[[1, 7]] @ w.t() + b, atol=1e-6) and float(out[0].abs().sum()) == 0
    a = torch.rand(6, 3) + 0.5; c = a.clone(); c[4, 1] += 1
    assert R.masked_isdiff(torch.tensor([0, 4, 5]), a, c, 1e-8, 1e-5).tolist() == [4]
    # quirk Q3 (main.cu:36): the tolerance uses the SIGNED `other`, so an unchanged row holding a value
    # below -atol/rtol is reported as different
    a[0, 0] = -1.0; c[0, 0] = -1.0
    assert R.masked_isdiff(torch.tensor([0, 4, 5]), a, c, 1e-8, 1e-5).tolist() == [0, 4]


# ---------------------------------------------------------------------------------------------
# host logic + C-ABI surface
# ---------------------------------------------------------------------------------------------
def test_capi_exports_every_declared_symbol_of_abi_3():
    from dagr_b200 import _lib, build
    so = build.build()
    lib = ctypes.CDLL(str(so))
    header = (ROOT / "include" / "dagr_b200.h").read_text()
    declared = set(re.findall(r"\b(dagr_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/dagr_b200.h but not exported"
    assert set(_lib.EXPORTS) == declared
    assert lib.dagr_abi_version() == 3


def test_product_has_no_cpu_fallback_and_never_imports_oracle():
    for p in (ROOT / "dagr_b200").rglob("*.py"):
        txt = p.read_text()
        assert "import oracle" not in txt and "from oracle" not in txt, p
    model, args = make_model("n", 180, 240)
    raw, data = make_inputs(1, 100, 240, 180)
    with pytest.raises(RuntimeError):
        model(data)                                  # CPU tensors: must fail loudly


def test_state_dict_layout_and_ema_deepcopy():
    from dagr_b200.model.ema import ModelEMA
    model, args = make_model("s")
    sd = model.state_dict()
    for k in ("backbone.conv_block1.conv_block1.conv.weight", "backbone.conv_block1.conv_block2.lin.mlp.weight",
              "backbone.layer5.conv_block2.norm_skip.module.running_var", "head.stem1.conv.lin.weight",
              "head.cls_pred2.bias", "head.stems.0.conv.weight", "head.obj_preds.1.bias"):
        assert k in sd, k
    assert sd["backbone.conv_block1.conv_block1.conv.weight"].shape == (25, 3, 16)
    assert sd["backbone.layer2.conv_block1.conv.weight"].shape == (25, 18, 64)
    assert sd["head.cls_pred1.weight"].shape == (25, 64, 2)
    ema = ModelEMA(model)
    ema.ema.load_state_dict(sd, strict=True)
    model.cache_luts(radius=args.radius, height=480, width=640)
    assert model.backbone.layer2.conv_block1.conv.lut_params["rx"] == 23


def test_yaml_config_surface():
    from dagr_b200.utils.args import FLAGS
    a = FLAGS(["--config", str(ROOT / "config" / "dagr-s-dsec.yaml"), "--batch_size", "8", "--use_image"])
    assert a.batch_size == 8 and a.net_stem_width == 0.5 and a.use_image and a.radius == 0.01


def test_oracle_full_forward_runs_and_is_deterministic():
    model, args = make_model("n", 180, 240, dataset="ncaltech101")
    raw, data = make_inputs(1, 3000, 240, 180, seed=3)
    from oracle.ref_model import RefModel
    ref = RefModel(model.state_dict(), args, 180, 240)
    o1 = ref.forward(data.x, data.pos, data.batch, 1)
    o2 = ref.forward(data.x, data.pos, data.batch, 1)
    assert torch.equal(o1["decoded"], o2["decoded"]) and o1["decoded"].shape == (1, 35, 105)
    # LUT path vs basis path agree (SURVEY 8c "extra internal checks")
    ref_b = RefModel(model.state_dict(), args, 180, 240, use_lut=False)
    o3 = ref_b.forward(data.x, data.pos, data.batch, 1)
    assert_close(o3["x1"], o1["x1"], tol=1e-3, what="basis vs LUT layer-1")


def test_oracle_reproduces_committed_golden_forward():
    """tests/golden/forward_dagr_n_240x180.pt (made by tests/golden/make_forward_golden.py) is reproduced bit for bit by
    the oracle on this machine: seeds, weights and the CPU restatement are stable."""
    from oracle.ref_model import RefModel
    fix = torch.load(GOLD / "forward_dagr_n_240x180.pt")
    m = fix["meta"]
    model, args = make_model(m["size"], m["H"], m["W"], seed=m["model_seed"])
    cs = float(sum(v.double().abs().sum() for v in model.state_dict().values() if v.dtype.is_floating_point))
    assert abs(cs - fix["weight_checksum"]) <= 1e-6 * abs(cs)
    o = RefModel(model.state_dict(), args, m["H"], m["W"]).forward(fix["x"], fix["pos"], fix["batch"], m["B"])
    assert torch.equal(o["edge_index"].int(), fix["edge_index"])
    assert torch.allclose(o["decoded"], fix["decoded"], rtol=1e-6, atol=1e-6)
    assert [len(d["boxes"]) for d in o["detections"]] == fix["n_det"]


def test_ingest_oracle_vs_reference_golden():
    """oracle/ref_ingest.py against tests/golden/downsample_golden.npz, which was produced by the reference's own numba
    down-sampler (scripts/downsample_events.py:91-124) with the change map carried over each case's chunks: every case,
    the seeded maps near +-1 at denominators 1, 2, 3, 8 and 9 included."""
    import numpy as np
    from pathlib import Path
    from oracle import ref_ingest as R
    from tests.helpers import downsample_golden_cases
    g = np.load(Path(__file__).parent / "golden" / "downsample_golden.npz")
    cases = downsample_golden_cases(g)
    assert len(cases) >= 10
    for case, (iw, ih, ow, oh), cm, chunks in cases:
        for k in range(chunks):
            ev = {q: g[f"c{case}_k{k}_in_{q}"] for q in "xypt"}
            out, cm = R.downsample_events(ev, ih, iw, oh, ow, change_map=cm)
            for q in "xypt":
                assert np.array_equal(out[q], g[f"c{case}_k{k}_out_{q}"]), (case, k, q)
            assert np.array_equal(cm, g[f"c{case}_k{k}_map"])


def test_ingest_window_oracle_identities():
    """dsec_data.py:141-147 + format/denormalise round trip: crop, window cut, t relative to the last kept event."""
    import numpy as np
    from oracle import ref_ingest as R
    rng = np.random.default_rng(3)
    n, W, H, T = 4000, 640, 430, 1_000_000
    ev = dict(x=rng.integers(0, W, n).astype("uint16"), y=rng.integers(0, 480, n).astype("uint16"),
              t=np.sort(rng.integers(10_000_000, 10_050_000, n)).astype("int64"), p=rng.integers(0, 2, n).astype("uint8"))
    den, pol = R.preprocess_window(ev, W, H, T, t_cut=10_040_000)
    keep = (ev["t"] < 10_040_000) & (ev["y"] < H)
    assert len(den) == int(keep.sum()) and set(np.unique(pol)) <= {-1.0, 1.0}
    assert np.array_equal(den[:, 0], ev["x"][keep]) and np.array_equal(den[:, 1], ev["y"][keep])
    t_rel = T + ev["t"][keep] - ev["t"][keep][-1]
    assert np.all(np.abs(den[:, 2] - t_rel) <= 1) and den[-1, 2] in (T, T - 1)       # fp32 round trip may lose 1 us
    den0, pol0 = R.preprocess_window({k: v[:0] for k, v in ev.items()}, W, H, T)
    assert den0.shape == (0, 3) and pol0.shape == (0,)


def test_detection_records_match_the_reference_golden(tmp_path):
    """dagr_b200.utils.buffers (host-side detection records, SURVEY 8(f)-2) against arrays produced by the reference's
    own src/dagr/utils/buffers.py (tests/golden/make_records_golden.py)."""
    import numpy as np
    from pathlib import Path
    from dagr.utils import buffers as B                      # the drop-in import path of the reference
    g = np.load(Path(__file__).parent / "golden" / "records_golden.npz")
    dets = [dict(boxes=torch.from_numpy(g[f"det{i}_boxes"]), scores=torch.from_numpy(g[f"det{i}_scores"]),
                 labels=torch.from_numpy(g[f"det{i}_labels"])) for i in range(4)]
    gts = [dict(boxes=torch.from_numpy(g[f"gt{i}_boxes"]), labels=torch.from_numpy(g[f"gt{i}_labels"])) for i in range(4)]
    seqs, ts = ["zurich_a", "zurich_a", "interlaken_b", "zurich_a"], [1000, 51000, 7, 101000]
    cd, cg = B.compile(dets, seqs, ts), B.compile(gts, seqs, ts)                 # DetectionBuffer.compile, buffers.py:112-115
    for s in ("zurich_a", "interlaken_b"):
        assert cd[s].dtype == g[f"compiled_det_{s}"].dtype and np.array_equal(cd[s], g[f"compiled_det_{s}"])
        assert cg[s].dtype == g[f"compiled_gt_{s}"].dtype and np.array_equal(cg[s], g[f"compiled_gt_{s}"])
    # run_test_interframe's to_npy / save_detections and the batched device form give the same records
    recs = [B.to_npy(dict(boxes=d["boxes"].numpy(), labels=d["labels"].numpy(), scores=d["scores"].numpy(), t=t)) for d, t in zip(dets, ts)]
    for r, d, t in zip(recs, dets, ts):
        ref = B.bbox_t_to_ndarray(d, t)
        assert r.dtype == ref.dtype and np.array_equal(r, ref)
    saved = B.save_detections(tmp_path, [dict(boxes=d["boxes"].numpy(), labels=d["labels"].numpy(), scores=d["scores"].numpy(), t=t, sequence=s)
                                         for d, t, s in zip(dets, ts, seqs)])
    assert np.array_equal(np.load(tmp_path / "detections_zurich_a.npy"), saved["zurich_a"])
    assert np.all(np.diff(saved["zurich_a"]["t"].astype(np.int64)) >= 0) and len(saved["zurich_a"]) == 8 and len(saved["interlaken_b"]) == 7
    A = 8
    det = torch.zeros(4, A, 6)
    ndet = torch.tensor([len(d["boxes"]) for d in dets], dtype=torch.int32)
    for b, d in enumerate(dets):
        n = len(d["boxes"])
        det[b, :n, :4], det[b, :n, 4], det[b, :n, 5] = d["boxes"], d["scores"], d["labels"].float()
    for r, ref in zip(B.records_from_device(det, ndet, ts), recs):
        assert r.dtype == ref.dtype and np.array_equal(r, ref)




def test_capi_check_config_and_workspace_sizes():
    """dagr_check_config states every kernel restriction in one call; *_workspace_bytes lets a foreign caller size buffers."""
    import ctypes as C
    from dagr_b200 import _lib
    from dagr_b200.geometry import Geometry
    lib = _lib.load()
    geom = Geometry(640, 480, 8, device="cpu")
    g = C.byref(geom.c_geom)
    assert lib.dagr_check_config(g, 2_400_000, 3, 16, b"relu") == 0
    assert lib.dagr_check_config(g, 2_400_000, 19, 16, None) == 0
    for bad, needle in (((g, 1 << 24, 3, 16, b"relu"), "24 bits"), ((g, 10, 5, 16, b"relu"), "conv_block1"), ((g, 10, 3, 32, b"relu"), "conv_block1"),
                        ((g, 10, 3, 16, b"elu"), "relu")):
        assert lib.dagr_check_config(*bad) == -3
        assert needle in lib.dagr_last_error().decode()
    big = Geometry(640, 480, 8, device="cpu")
    big.c_geom.K = 17
    assert lib.dagr_check_config(C.byref(big.c_geom), 10, 3, 16, b"relu") == -3 and "max_neighbors" in lib.dagr_last_error().decode()
    N = 2_400_000
    sz = _lib.EventWs()
    assert lib.dagr_event_workspace_bytes(g, N, C.byref(sz)) == 0
    cells = 8 * 56 * 40
    assert (sz.key, sz.perm, sz.ti, sz.nbr, sz.off, sz.xa) == (4 * N, 4 * N, 8 * N, 64 * N, 32 * N, 64 * N)
    assert sz.start == 4 * (geom.NK + 1) and sz.count == sz.start and sz.cellmask == 4 * cells and sz.wl_ids == 4 * cells
    assert sz.blocksums == 4 * (int(lib.dagr_scan_blocks(max(geom.NK + 1, N + 1))) + 2)
    ps = _lib.PoolWs()
    assert lib.dagr_pool_workspace_bytes(8 * 28 * 20, 64, C.byref(ps)) == 0
    assert (ps.acc, ps.possum, ps.pcnt) == (8 * 28 * 20 * 64 * 8, 8 * 28 * 20 * 24, 8 * 28 * 20 * 4)
