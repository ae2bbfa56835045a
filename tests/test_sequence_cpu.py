"""Detection over a recorded sequence without a GPU: the argument contract of dagr_window_bounds and dagr_window_gather
(every bad input is refused with DAGR_E_ARG and a message naming the function before anything is launched), the block
planner, interframe_windows against the reference script's loop, and SequenceDetector's constructor and input checks
(all of them raise before any device work)."""
import ctypes as C

import numpy as np
import pytest

from tests.helpers import make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first
W, H = 320, 215


def _bounds(lib, t=BAD, N=10, tb=BAD, te=BAD, Q=4, begin=BAD, end=BAD):
    return lib.dagr_window_bounds(t, N, tb, te, Q, begin, end, None)


def _gather(lib, x=BAD, y=BAD, t=BAD, p=BAD, N=10, begin=BAD, end=BAD, G=4, t_base=0, p01=1, total=100, batch=BAD, pos=BAD,
            feat=BAD, offs=BAD):
    return lib.dagr_window_gather(x, y, t, p, N, begin, end, G, t_base, p01, total, batch, pos, feat, offs, None)


@pytest.mark.parametrize("fn,kw,needle", [
    ("dagr_window_bounds", dict(t=None), "null t"),
    ("dagr_window_bounds", dict(tb=None), "null"),
    ("dagr_window_bounds", dict(te=None), "null"),
    ("dagr_window_bounds", dict(begin=None), "null"),
    ("dagr_window_bounds", dict(end=None), "null"),
    ("dagr_window_bounds", dict(N=-1), "N must"),
    ("dagr_window_bounds", dict(N=1 << 31), "N must"),
    ("dagr_window_bounds", dict(Q=-1), "Q must"),
    ("dagr_window_bounds", dict(Q=1 << 31), "Q must"),
    ("dagr_window_gather", dict(begin=None), "null"),
    ("dagr_window_gather", dict(end=None), "null"),
    ("dagr_window_gather", dict(offs=None), "null"),
    ("dagr_window_gather", dict(x=None), "null"),
    ("dagr_window_gather", dict(t=None), "null"),
    ("dagr_window_gather", dict(p=None), "null"),
    ("dagr_window_gather", dict(batch=None), "null"),
    ("dagr_window_gather", dict(pos=None), "null"),
    ("dagr_window_gather", dict(feat=None), "null"),
    ("dagr_window_gather", dict(N=-1), "N must"),
    ("dagr_window_gather", dict(N=1 << 31), "N must"),
    ("dagr_window_gather", dict(G=0), "G must"),
    ("dagr_window_gather", dict(G=256), "G must"),
    ("dagr_window_gather", dict(total=-1), "block total"),
    ("dagr_window_gather", dict(total=1 << 24), "block total"),
])
def test_window_entry_points_reject_bad_arguments(fn, kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    call = _bounds if fn == "dagr_window_bounds" else _gather
    assert call(lib, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert fn in msg and needle in msg, msg


def test_window_bounds_without_windows_launches_nothing():
    """Q = 0 (and N = 0): every row may be NULL and the call returns before touching the device."""
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _bounds(lib, t=None, N=0, tb=None, te=None, Q=0, begin=None, end=None) == 0


# ---- block planning ---------------------------------------------------------------------------------------------------
def _check_plan(sizes, mw, me):
    from dagr_b200.sequence import plan_blocks
    blocks = plan_blocks(sizes, mw, me)
    assert [q for b in blocks for q in range(*b)] == list(range(len(sizes)))       # every window once, in order
    for q0, q1 in blocks:
        assert 1 <= q1 - q0 <= mw
        tot = int(np.sum(sizes[q0:q1]))
        assert tot <= me or q1 - q0 == 1                                           # only a lone window may exceed max_events
    for (a0, a1), (b0, b1) in zip(blocks, blocks[1:]):                             # greedy: the next window did not fit
        assert a1 - a0 == mw or int(np.sum(sizes[a0:a1 + 1])) > me
    return blocks


def test_plan_respects_max_windows_and_max_events():
    rng = np.random.default_rng(0)
    sizes = rng.integers(0, 60_000, 500)
    sizes[::37] = 0
    for mw in (1, 7, 64, 255):
        for me in (1, 50_000, 400_000, 1 << 23):
            _check_plan(sizes, mw, me)
    assert len(_check_plan(sizes, 255, 1 << 23)) == 2                              # 500 windows, well under the event cap


def test_plan_runs_an_oversized_window_alone_and_refuses_2_24():
    from dagr_b200.sequence import plan_blocks
    sizes = np.array([10, 20, 500, 30, 40, 0, 600, 5])
    assert plan_blocks(sizes, 64, 100) == [(0, 2), (2, 3), (3, 6), (6, 7), (7, 8)]
    assert plan_blocks([(1 << 24) - 1], 8, 10) == [(0, 1)]
    assert plan_blocks([], 8, 10) == []
    with pytest.raises(ValueError, match="2\\^24"):
        plan_blocks([5, 1 << 24, 3], 64, 1 << 23)


# ---- interframe windows -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("steps,span", [(10, 50_000), (7, 50_000), (3, 33_333), (1, 50_000)])
def test_interframe_windows_equal_the_script_loop(steps, span):
    """scripts/run_test_interframe.py: `for n_us in np.linspace(0, 50000, steps)` re-runs the test set with windows
    [frame t, frame t + int(n_us)), offset-major."""
    from dagr_b200.sequence import interframe_windows
    frame_t = np.array([0, 50_000, 100_000, 150_123, 400_000], dtype=np.int64) + 7_000_000_000
    want = [(int(ft), int(ft) + int(n_us), i) for n_us in np.linspace(0, span, steps) for i, ft in enumerate(frame_t)]
    tb, te, fi = interframe_windows(frame_t, steps=steps, span_us=span)
    assert tb.dtype == te.dtype == fi.dtype == np.int64
    assert list(zip(tb.tolist(), te.tolist(), fi.tolist())) == want
    assert (te[:len(frame_t)] == tb[:len(frame_t)]).all()                          # the first window of each frame is empty


# ---- constructor and input checks -------------------------------------------------------------------------------------
def _events(n=100, seed=0):
    rng = np.random.default_rng(seed)
    return dict(x=rng.integers(0, W, n).astype(np.int16), y=rng.integers(0, H, n).astype(np.int16),
                t=np.sort(rng.integers(0, 100_000, n)).astype(np.int32), p=rng.choice([-1, 1], n).astype(np.int8))


@pytest.fixture(scope="module")
def events_model():
    return make_model("s", H, W)[0]


@pytest.fixture(scope="module")
def hybrid_model():
    return make_model("s", H, W, use_image=True, img_net="resnet18")[0]


def test_constructor_refusals(events_model, hybrid_model):
    from dagr_b200.sequence import SequenceDetector
    with pytest.raises(ValueError, match="raw_frames"):
        SequenceDetector(hybrid_model, raw_frames=True)
    with pytest.raises(ValueError, match="image-fusion"):
        SequenceDetector(events_model, sensor=(640, 480), raw_frames=True)
    with pytest.raises(ValueError, match="max_windows"):
        SequenceDetector(events_model, max_windows=256)
    with pytest.raises(ValueError, match="max_windows"):
        SequenceDetector(events_model, max_windows=0)
    with pytest.raises(ValueError, match="max_events"):
        SequenceDetector(events_model, max_events=1 << 24)
    with pytest.raises(ValueError, match="p_is_01"):
        SequenceDetector(events_model, p_is_01=False)
    with pytest.raises(ValueError, match="sensor"):
        SequenceDetector(events_model, sensor=(500, 480))
    no_events = make_model("n", H, W, use_image=True, no_events=True, img_net="resnet18")[0]
    with pytest.raises(NotImplementedError, match="no_events"):
        SequenceDetector(no_events)
    assert SequenceDetector(hybrid_model).image_precision == hybrid_model.image_precision


def test_input_checks_raise_before_device_work(events_model, hybrid_model):
    from dagr_b200.sequence import SequenceDetector
    det = SequenceDetector(events_model)
    ev = _events()
    bad = dict(ev, t=ev["t"][::-1].copy())
    with pytest.raises(ValueError, match="sorted"):
        det.detect(bad, [50_000])
    with pytest.raises(ValueError, match="lengths"):
        det.detect(dict(ev, p=ev["p"][:-1]), [50_000])
    with pytest.raises(ValueError, match="x, y, t and p"):
        det.detect(dict(x=ev["x"], y=ev["y"], t=ev["t"]), [50_000])
    with pytest.raises(ValueError, match="int32"):
        det.detect(dict(ev, t=ev["t"].astype(np.int64) + (1 << 31)), [50_000])
    with pytest.raises(ValueError, match="t_begin"):
        det.detect(ev, [50_000, 60_000], t_begin=[0])
    with pytest.raises(ValueError, match="t_begin > t_end"):
        det.detect(ev, [50_000], t_begin=[50_001])
    with pytest.raises(ValueError, match="events-only"):
        det.detect(ev, [50_000], frames=np.zeros((1, 3, H, W), np.uint8), frame_t=[0])
    raw = SequenceDetector(events_model, sensor=(640, 480))
    with pytest.raises(ValueError, match="sensor"):
        raw.detect(dict(ev, x=ev["x"].astype(np.int64) + 600), [50_000])
    with pytest.raises(ValueError, match="polarities"):
        raw.detect(ev, [50_000])                                                   # +-1 with p_is_01=True
    fus = SequenceDetector(hybrid_model)
    frames = np.zeros((2, 3, H, W), np.uint8)
    with pytest.raises(ValueError, match="before the first frame"):
        fus.detect(ev, [60_000, 20_000], frames=frames, frame_t=[30_000, 60_000])
    with pytest.raises(ValueError, match="needs frames"):
        fus.detect(ev, [60_000])
    with pytest.raises(ValueError, match="frame_t"):
        fus.detect(ev, [60_000], frames=frames)
    with pytest.raises(ValueError, match="frame times"):
        fus.detect(ev, [60_000], frames=frames, frame_t=[0])
    with pytest.raises(ValueError, match="frame indices"):
        fus.detect(ev, [60_000], frames=frames, frame_idx=[2])
    with pytest.raises(ValueError, match="frame of shape"):
        fus.detect(ev, [60_000], frames=np.zeros((2, 3, H, W + 1), np.uint8), frame_t=[0, 10])
    # valid input on a CPU model gets as far as the device check
    with pytest.raises(RuntimeError, match="CUDA"):
        det.detect(ev, [50_000, 10_000])
