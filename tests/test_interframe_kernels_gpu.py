"""The interframe evaluation kernels (csrc/labels.cu) on their own: dagr_interframe_targets equals the oracle's NumPy-1 rule
(oracle/ref_labels.py) bit for bit on the golden recordings and on random tables of up to 10^5 windows, and
dagr_eval_pack_detections equals a numpy packing of det / ndet; bad shapes return the C-ABI error."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest
import torch

from dagr_b200 import _lib
from dagr_b200 import labels as L
from oracle import ref_labels as R

pytestmark = pytest.mark.gpu

Z = np.load(Path(__file__).parent / "golden" / "interframe_labels_golden.npz")
W, H, SCALE, MIN_H, MIN_D = (int(v) for v in Z["dims"])
K = 2


def d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_targets(box0, box1, cls, off, pair_t, win_pair, win_t, win_group, width=W, height=H, min_h=MIN_H, min_d=MIN_D, fill=0x7F):
    lib = _lib.load()
    off = np.asarray(off, np.int64)
    Q = len(win_pair)
    R_ = int((off[np.asarray(win_pair) + 1] - off[np.asarray(win_pair)]).sum()) if Q else 0
    need = C.c_int64(0)
    _lib.check(lib.dagr_interframe_targets_workspace_bytes(Q, R_, C.byref(need)))
    ws = torch.full((need.value,), fill, dtype=torch.uint8, device="cuda")
    gt_box = torch.full((max(R_, 1), 4), -7.0, device="cuda")
    gt_label = torch.full((max(R_, 1),), -7, dtype=torch.int64, device="cuda")
    gt_off = torch.full((Q + 1,), -7, dtype=torch.int64, device="cuda")
    args = [d(np.asarray(box0, np.float32).reshape(-1, 4)), d(np.asarray(box1, np.float32).reshape(-1, 4)), d(np.asarray(cls, np.int64)),
            d(off), d(np.asarray(pair_t, np.int64).reshape(-1)), d(np.asarray(win_pair, np.int64)), d(np.asarray(win_t, np.int64)),
            d(np.asarray(win_group, np.int32))]
    _lib.check(lib.dagr_interframe_targets(*[_lib.ptr(a) for a in args[:5]], len(off) - 1, len(box0), *[_lib.ptr(a) for a in args[5:]], Q, K,
                                           width, height, float(min_h), float(min_d), R_, _lib.ptr(ws), ws.numel(), _lib.ptr(gt_box),
                                           _lib.ptr(gt_label), _lib.ptr(gt_off), _lib.stream_ptr()), "dagr_interframe_targets")
    o = gt_off.cpu().numpy()
    n = int(o[-1])
    return gt_box.cpu().numpy()[:n], gt_label.cpu().numpy()[:n], o, gt_box.cpu().numpy()[n:R_]


def check_targets(*tables, **kw):
    got = run_targets(*tables, **kw)
    want = R.flat_targets(*tables, K, kw.get("width", W), kw.get("height", H), kw.get("min_h", MIN_H), kw.get("min_d", MIN_D))
    assert got[0].shape == want[0].shape and np.array_equal(got[0].view(np.int32), want[0].view(np.int32))
    assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
    assert (got[3] == -7.0).all()                                              # nothing written past the kept rows
    return want


@pytest.mark.parametrize("name", ["rec_a", "rec_b"])
def test_targets_equal_the_reference_on_the_golden_recordings(name):
    pl = L.pair_labels(Z[f"{name}_tracks"], Z[f"{name}_image_ts"], tuple(str(s) for s in Z["source"]), W, H, SCALE, MIN_H, MIN_D)
    offs = [int(v) for v in Z["offsets"]]
    P = len(pl)
    win_t = (pl.t[:, 0][None, :] + np.array(offs)[:, None]).reshape(-1)
    group = np.repeat(np.arange(len(offs)), P)
    box, lab, off, _ = run_targets(pl.box0, pl.box1, pl.cls, pl.off, pl.t, np.tile(np.arange(P), len(offs)), win_t, group)
    assert np.array_equal(box.view(np.int32), Z[f"{name}_numpy1_box"].view(np.int32))        # the reference itself
    assert np.array_equal(off, Z[f"{name}_numpy1_off"])
    assert np.array_equal(lab, np.repeat(group, np.diff(off)) * K + Z[f"{name}_numpy1_label"])


def random_tables(rng, P, rows_max, empty_frac=0.1):
    n = rng.integers(0, rows_max + 1, P)
    n[rng.random(P) < empty_frac] = 0
    off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    Lr = int(off[-1])
    xy0 = rng.uniform(-60, 360, (Lr, 2))
    wh0 = rng.uniform(0, 90, (Lr, 2))
    b0 = np.concatenate([xy0, wh0], 1).astype(np.float32)
    b1 = (b0 + rng.normal(0, 15, (Lr, 4))).astype(np.float32)
    t0 = rng.integers(0, 1 << 40, P)
    pair_t = np.stack([t0, t0 + rng.integers(1, 60_000, P)], 1)
    return b0, b1, rng.integers(0, K, Lr), off, pair_t


@pytest.mark.parametrize("Q", [1, 1000, 100_000])
def test_targets_equal_the_oracle_on_random_tables(Q):
    rng = np.random.default_rng(Q)
    P = max(Q // 10, 1)
    b0, b1, cls, off, pair_t = random_tables(rng, P, 12)
    win_pair = rng.integers(0, P, Q)
    win_t = pair_t[win_pair, 0] + rng.integers(0, 70_000, Q)                   # r in [0, > 1)
    win_t[::7] = pair_t[win_pair[::7], 0]                                      # r = 0
    win_t[3::7] = pair_t[win_pair[3::7], 1]                                    # r = 1
    want = check_targets(b0, b1, cls, off, pair_t, win_pair, win_t, rng.integers(0, 10, Q))
    assert Q < 1000 or 0 < len(want[0]) < int((off[win_pair + 1] - off[win_pair]).sum())  # some rows kept, some filtered


def test_targets_edge_windows():
    rng = np.random.default_rng(5)
    b0, b1, cls, off, pair_t = random_tables(rng, 6, 40, empty_frac=0)
    off = np.array([0, 0, off[2], off[2], off[4], off[4], off[6]])             # pairs 0, 2 and 4 are empty
    pair_t = np.concatenate([pair_t, pair_t[:1]])
    b0[off[4]:off[6], 2:] = 3.0                                                # pair 5: every row below the size filter
    b1[off[4]:off[6], 2:] = 3.0
    win_pair = np.array([0, 1, 2, 3, 4, 5, 5, 0, 1])
    win_t = pair_t[win_pair, 0] + 20_000
    out = check_targets(b0, b1, cls, off, pair_t, win_pair, win_t, np.arange(9) % 3)
    assert np.diff(out[2])[[0, 2, 4, 5, 6, 7]].tolist() == [0] * 6
    # one window holding every row, at r = 0 (the frame's own boxes)
    one = np.array([0, len(b0)])
    check_targets(b0, b1, cls, one, pair_t[:1], [0], [pair_t[0, 0]], [0])
    check_targets(b0, b1, cls, one, pair_t[:1], [0, 0], [pair_t[0, 1], pair_t[0, 0] + 7], [3, 1])
    # no window at all
    got = run_targets(b0, b1, cls, off, pair_t, np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int32))
    assert got[2].tolist() == [0]


def pack_numpy(det, ndet, group, gt_off, K):
    Q, A, _ = det.shape
    has_gt = np.diff(gt_off) > 0
    n = np.where(has_gt, np.clip(ndet, 0, A), 0)
    rows = np.concatenate([det[q, :n[q]] for q in range(Q)]) if Q else np.zeros((0, 6), np.float32)
    g = np.repeat(np.asarray(group, np.int64), n)
    lab = rows[:, 5]
    label = np.where((lab >= 0) & (lab < K), g * K + lab.astype(np.int64), -1)
    return rows[:, :4].copy(), rows[:, 4].copy(), label, np.concatenate([[0], np.cumsum(n)]).astype(np.int64)


def run_pack(det, ndet, group, gt_off):
    lib = _lib.load()
    Q, A, _ = det.shape
    need = C.c_int64(0)
    _lib.check(lib.dagr_eval_pack_workspace_bytes(Q, C.byref(need)))
    ws = torch.full((need.value,), 0xFF, dtype=torch.uint8, device="cuda")
    dt_box = torch.full((max(Q * A, 1), 4), -7.0, device="cuda")
    dt_score = torch.full((max(Q * A, 1),), -7.0, device="cuda")
    dt_label = torch.full((max(Q * A, 1),), -7, dtype=torch.int64, device="cuda")
    dt_off = torch.empty(Q + 1, dtype=torch.int64, device="cuda")
    dd, dn, dg, do = d(det), d(ndet.astype(np.int32)), d(np.asarray(group, np.int32)), d(gt_off)
    _lib.check(lib.dagr_eval_pack_detections(_lib.ptr(dd), _lib.ptr(dn), Q, A, _lib.ptr(dg), _lib.ptr(do), K, _lib.ptr(ws), ws.numel(),
                                             _lib.ptr(dt_box), _lib.ptr(dt_score), _lib.ptr(dt_label), _lib.ptr(dt_off), _lib.stream_ptr()),
               "dagr_eval_pack_detections")
    o = dt_off.cpu().numpy()
    n = int(o[-1])
    return dt_box.cpu().numpy()[:n], dt_score.cpu().numpy()[:n], dt_label.cpu().numpy()[:n], o


@pytest.mark.parametrize("Q,A", [(1, 1), (37, 100), (20_000, 100)])
def test_pack_equals_numpy(Q, A):
    rng = np.random.default_rng(Q + A)
    det = rng.normal(100, 50, (Q, A, 6)).astype(np.float32)
    det[..., 5] = rng.integers(0, K, (Q, A))
    det[0, :, 5] = 5.0 if Q > 1 else det[0, :, 5]                              # a label outside [0, K): no category
    ndet = rng.integers(0, A + 1, Q)
    ndet[::5] = 0
    ndet[1::5] = A
    gt_n = rng.integers(0, 3, Q)                                               # a third of the windows without GT
    gt_off = np.concatenate([[0], np.cumsum(gt_n)]).astype(np.int64)
    group = rng.integers(0, 10, Q)
    got, want = run_pack(det, ndet, group, gt_off), pack_numpy(det, ndet, group, gt_off, K)
    for g, w in zip(got, want):
        assert g.shape == w.shape and np.array_equal(g.view(np.int32) if g.dtype == np.float32 else g, w.view(np.int32) if w.dtype == np.float32 else w)
    assert (np.diff(got[3])[gt_n == 0] == 0).all()


def test_bad_shapes_return_the_abi_error():
    lib = _lib.load()
    out = C.c_int64(0)
    assert lib.dagr_interframe_targets_workspace_bytes(-1, 0, C.byref(out)) == -1
    assert lib.dagr_interframe_targets_workspace_bytes(1, 1 << 31, C.byref(out)) == -1
    assert lib.dagr_eval_pack_workspace_bytes(-1, C.byref(out)) == -1
    assert lib.dagr_eval_pack_workspace_bytes(5, None) == -1
    ws = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    buf = torch.empty(1 << 12, dtype=torch.float32, device="cuda")
    p, s = _lib.ptr(buf), _lib.stream_ptr()
    # K = 0; windows without a pair to refer to; a workspace that is too small; a misaligned box array
    assert lib.dagr_interframe_targets(p, p, p, p, p, 1, 1, p, p, p, 1, 0, W, H, 10.0, 15.0, 1, _lib.ptr(ws), ws.numel(), p, p, p, s) == -1
    assert lib.dagr_interframe_targets(p, p, p, p, p, 0, 1, p, p, p, 1, K, W, H, 10.0, 15.0, 1, _lib.ptr(ws), ws.numel(), p, p, p, s) == -1
    assert lib.dagr_interframe_targets(p, p, p, p, p, 1, 1, p, p, p, 1, K, W, H, 10.0, 15.0, 1, _lib.ptr(ws), 16, p, p, p, s) == -1
    odd = C.c_void_p(buf.data_ptr() + 4)
    assert lib.dagr_interframe_targets(odd, p, p, p, p, 1, 1, p, p, p, 1, K, W, H, 10.0, 15.0, 1, _lib.ptr(ws), ws.numel(), p, p, p, s) == -1
    assert lib.dagr_interframe_targets(p, p, p, p, p, 1, 1, p, p, p, 1, K, 0, H, 10.0, 15.0, 1, _lib.ptr(ws), ws.numel(), p, p, p, s) == -1
    assert lib.dagr_interframe_targets(p, p, p, p, p, 1, 1, None, p, p, 1, K, W, H, 10.0, 15.0, 1, _lib.ptr(ws), ws.numel(), p, p, p, s) == -1
    # A = 0; Q * A past 2^31; null outputs; a workspace that is too small
    assert lib.dagr_eval_pack_detections(p, p, 1, 0, p, p, K, _lib.ptr(ws), ws.numel(), p, p, p, p, s) == -1
    assert lib.dagr_eval_pack_detections(p, p, 1 << 25, 100, p, p, K, _lib.ptr(ws), ws.numel(), p, p, p, p, s) == -1
    assert lib.dagr_eval_pack_detections(p, p, 1, 1, p, p, K, _lib.ptr(ws), ws.numel(), None, p, p, p, s) == -1
    assert lib.dagr_eval_pack_detections(p, p, 1, 1, p, p, K, _lib.ptr(ws), 8, p, p, p, p, s) == -1
    assert b"dagr_eval_pack_detections" in lib.dagr_last_error()
    torch.cuda.synchronize()                                                   # nothing was launched
