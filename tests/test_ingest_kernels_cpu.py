"""The batch event ingest without a GPU: oracle/ref_ingest.preprocess_window against the reference's own preprocessing
chain (tests/golden/ingest_window_golden.npz: DSEC.preprocess_events, to_data, format_data and denormalize_pos run
unmodified), bit for bit, on the window edge cases and on the exhaustive denormalisation sweep; and the argument contract
of dagr_downsample_events, dagr_compact_events and dagr_ingest_events (every bad input is refused with DAGR_E_ARG and a
message naming the function before anything is launched)."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first
WINDOW_GOLD = Path(__file__).resolve().parent / "golden" / "ingest_window_golden.npz"
NCASES = 11


def window_case(g, i):
    """case i of the window fixture -> (events dict, W, H, T, t_cut, reference pos, reference feat)."""
    ev = {k: g[f"c{i}_in_{k}"] for k in "xytp"}
    W, H, T = (int(v) for v in g[f"c{i}_dims"])
    return ev, W, H, T, int(g[f"c{i}_t_cut"]), g[f"c{i}_pos"], g[f"c{i}_feat"]


def sweep_events(W, H, T, base=0):
    """the sweep window of (W, H, T): T + 1 sorted events with relative t = 0..T, x = i % W, y = i % H, p = i & 1."""
    i = np.arange(T + 1, dtype=np.int64)
    return dict(x=(i % W).astype(np.uint16), y=(i % H).astype(np.uint16), t=i + base, p=(i & 1).astype(np.uint8))


def sweep_expected(g, W, H, T):
    """the reference's denormalised (x, y, t) of sweep_events(W, H, T): the input, except at the stored coordinates."""
    i = np.arange(T + 1, dtype=np.int64)
    cols = []
    for name, dim, v in (("x", W, i % W), ("y", H, i % H), ("t", T, i)):
        lut = np.arange(dim + 1, dtype=np.int32)
        lut[g[f"sweep_{name}{dim}_in"]] = g[f"sweep_{name}{dim}_out"]
        cols.append(lut[v])
    return np.stack(cols, 1)


@pytest.mark.parametrize("case", range(NCASES))
def test_preprocess_window_oracle_equals_reference_golden(case):
    from oracle import ref_ingest as R
    g = np.load(WINDOW_GOLD)
    ev, W, H, T, cut, pos, feat = window_case(g, case)
    den, pol = R.preprocess_window({k: v.copy() for k, v in ev.items()}, W, H, T, t_cut=cut)
    assert den.dtype == np.int32 and pol.dtype == np.float32
    assert np.array_equal(den, pos) and np.array_equal(pol, feat)


def test_window_golden_covers_its_edges():
    """the cases of the fixture are the edges they are named for."""
    g = np.load(WINDOW_GOLD)
    kept = []
    for i in range(NCASES):
        ev, W, H, T, cut, pos, feat = window_case(g, i)
        k = (ev["t"] < cut) & (ev["y"] < H)
        assert len(pos) == int(k.sum()) and set(np.unique(feat)) <= {-1.0, 1.0}
        kept.append(ev["t"][k])
    ev1, cut1 = window_case(g, 1)[0], window_case(g, 1)[4]
    assert (ev1["t"] == cut1).any() and (ev1["t"] == cut1 - 1).any()
    assert ((window_case(g, 2)[0]["y"] == 430).sum() >= 1) and ((window_case(g, 2)[0]["y"] == 429).sum() >= 1)
    ev3 = window_case(g, 3)[0]
    assert ev3["t"][-1] > kept[3][-1]                                    # the latest events are cropped away
    assert (kept[4] == kept[4][-1]).sum() > 1                            # a tie at the last event
    assert len(kept[5]) == 0
    assert kept[6].min() >= 1 << 32
    assert window_case(g, 7)[0]["x"].max() >= 1 << 15
    assert kept[8][-1] - kept[8][0] >= 1 << 32
    assert kept[9][-1] not in (kept[9].max(), kept[9].min()) and (np.diff(kept[9]) < 0).any()
    assert kept[10].max() < 0


def test_preprocess_window_oracle_equals_reference_sweep():
    """every t in [0, T] and every x < W, y < H of the fixture's sweep: the oracle denormalises each to the reference's
    value, which is the input except at the stored coordinates (only t at T = 10^6 and 999 999 truncates below)."""
    from oracle import ref_ingest as R
    g = np.load(WINDOW_GOLD)
    dims = [tuple(int(v) for v in d) for d in g["sweep_dims"]]
    assert len(dims) == 12
    for W, H, T in dims:
        den, pol = R.preprocess_window(sweep_events(W, H, T, base=7_000_000_000), W, H, T)
        assert np.array_equal(den, sweep_expected(g, W, H, T)), (W, H, T)
    assert len(g["sweep_t1000000_in"]) > 10_000 and len(g["sweep_t50000_in"]) == 0
    assert all(len(g[f"sweep_x{W}_in"]) == 0 for W in (640, 320, 240, 1280))


# ---------------------------------------------------------------------------------------------------------------------
# argument contract
# ---------------------------------------------------------------------------------------------------------------------
def _downsample(lib, x=BAD, y=BAD, p=BAD, N=100, fx=2, fy=2, ow=320, oh=240, cmap=BAD, cell=BAD, tmp=BAD, srt=BAD,
                count=BAD, start=BAD, bs=BAD, mask=BAD):
    return lib.dagr_downsample_events(x, y, p, N, fx, fy, ow, oh, cmap, cell, tmp, srt, count, start, bs, mask, None)


def _compact(lib, mask=BAD, N=100, x=BAD, y=BAD, t=BAD, p=BAD, fx=2, fy=2, flag=BAD, pos=BAD, bs=BAD, xo=BAD, yo=BAD,
             to=BAD, po=BAD, n_out=BAD):
    return lib.dagr_compact_events(mask, N, x, y, t, p, fx, fy, flag, pos, bs, xo, yo, to, po, n_out, None)


def _ingest(lib, x=BAD, y=BAD, t=BAD, p=BAD, N=100, W=640, H=430, T=1_000_000, flag=BAD, pos=BAD, bs=BAD, tlast=BAD,
            batch=BAD, pos_o=BAD, feat=BAD, n_out=BAD):
    return lib.dagr_ingest_events(x, y, t, p, N, 1, W, H, T, 1 << 62, 0, flag, pos, bs, tlast, batch, pos_o, feat, n_out, None)


CALLS = {"dagr_downsample_events": _downsample, "dagr_compact_events": _compact, "dagr_ingest_events": _ingest}


@pytest.mark.parametrize("fn,kw,needle", [
    ("dagr_downsample_events", dict(cmap=None), "null"),
    ("dagr_downsample_events", dict(count=None), "null"),
    ("dagr_downsample_events", dict(start=None), "null"),
    ("dagr_downsample_events", dict(bs=None), "null"),
    ("dagr_downsample_events", dict(x=None), "null"),
    ("dagr_downsample_events", dict(p=None), "null"),
    ("dagr_downsample_events", dict(srt=None), "null"),
    ("dagr_downsample_events", dict(mask=None), "null"),
    ("dagr_downsample_events", dict(N=-1), "N must"),
    ("dagr_downsample_events", dict(N=1 << 31), "N must"),
    ("dagr_downsample_events", dict(fx=0), "geometry"),
    ("dagr_downsample_events", dict(fy=-1), "geometry"),
    ("dagr_downsample_events", dict(ow=0), "geometry"),
    ("dagr_downsample_events", dict(oh=0), "geometry"),
    ("dagr_downsample_events", dict(ow=65536, oh=32768, fx=1, fy=1), "out_w * out_h"),
    ("dagr_compact_events", dict(pos=None), "null"),
    ("dagr_compact_events", dict(bs=None), "null"),
    ("dagr_compact_events", dict(n_out=None), "null"),
    ("dagr_compact_events", dict(mask=None), "null"),
    ("dagr_compact_events", dict(t=None), "null"),
    ("dagr_compact_events", dict(flag=None), "null"),
    ("dagr_compact_events", dict(po=None), "null"),
    ("dagr_compact_events", dict(N=-5), "N must"),
    ("dagr_compact_events", dict(N=1 << 31), "N must"),
    ("dagr_compact_events", dict(fx=0), "fx"),
    ("dagr_compact_events", dict(fy=0), "fx"),
    ("dagr_ingest_events", dict(pos=None), "null"),
    ("dagr_ingest_events", dict(bs=None), "null"),
    ("dagr_ingest_events", dict(tlast=None), "null"),
    ("dagr_ingest_events", dict(n_out=None), "null"),
    ("dagr_ingest_events", dict(t=None), "null"),
    ("dagr_ingest_events", dict(flag=None), "null"),
    ("dagr_ingest_events", dict(feat=None), "null"),
    ("dagr_ingest_events", dict(N=-1), "N must"),
    ("dagr_ingest_events", dict(N=1 << 31), "N must"),
    ("dagr_ingest_events", dict(W=0), "W, H and T"),
    ("dagr_ingest_events", dict(H=0), "W, H and T"),
    ("dagr_ingest_events", dict(T=0), "W, H and T"),
])
def test_batch_ingest_rejects_bad_arguments(fn, kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert CALLS[fn](lib, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert fn in msg and needle in msg, msg


def test_downsample_with_no_events_needs_no_rows():
    """N = 0: the N-long rows may be NULL, and nothing is launched (the call returns before touching the device)."""
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _downsample(lib, x=None, y=None, p=None, N=0, cell=None, tmp=None, srt=None, mask=None) == 0
