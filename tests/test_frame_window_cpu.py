"""Interframe windows on live hybrid cameras (since_frame=True), the host side without a GPU: the window rule t_cut =
max(t_us of the frame a step reads, t_end - window_us) on both time axes, the frame a step may read (never one later than
its t_end), the refusals raised before any device work, the cut stage of the second push and, through the host model of
the ring push, that the two pushes leave exactly the events of [t_cut, t_end)."""
import numpy as np
import pytest

from tests.helpers import make_model


class _Ready:
    def __init__(self, done):
        self.done = done

    def query(self):
        return self.done

    def synchronize(self):
        self.done = True


class _Stream:
    def wait_event(self, ev):
        pass


class _Det:
    """what _CameraFrames reads of its detector before any device work."""
    since_frame, raw_frames, W, H = True, False, 8, 6
    stream = _Stream()


def _cam(frames=(), cur=None):
    """a camera whose frame in use has time `cur` (None: no frame yet) and whose pending frame is `frames` = (t_us, done)."""
    from dagr_b200.streaming import _CameraFrames
    c = _CameraFrames(_Det(), 0)
    if cur is not None:
        c.cur, c.cur_frame, c.nframes = 0, (0, cur), 1
    for t_us, done in frames:
        c.pending = dict(slot=0 if c.cur is None else 1 - c.cur, id=c.nframes, t_us=t_us, ready=_Ready(done), trunk=None)
        c.nframes += 1
    return c


def test_cut_starts_at_the_frame_and_window_us_caps_it():
    W = 50_000
    c = _cam(cur=100_000)
    for te in (100_000, 101_000, 149_999, 150_000, 150_001, 400_000):
        take, cut = c.plan(te, te - W, 0)
        assert not take and cut == max(100_000, te - W), te
    # raw sensor time: the frame's raw time is rebased by the stream's time base like the chunks
    base = 7_000_000_000
    c = _cam(cur=base + 100_000)
    for te in (100_000, 120_000, 160_000):                           # rebased t_end
        assert c.plan(te + base, te - W, base) == (False, max(100_000, te - W)), te
    assert c.plan(base + 200_000, -2**31, None) == (False, -2**31)  # no time base yet: the ring is empty, the cut stands
    c = _cam(cur=base - 10)                                           # a frame before the stream's first event
    assert c.plan(base + 100, 100 - W, base) == (False, -10)
    c = _cam(cur=base + 2**31)
    with pytest.raises(ValueError, match="int32"):
        c.plan(base + 2**31 + 5, 2**31 - 1 - W, base)


def test_a_step_never_reads_a_frame_later_than_its_t_end():
    c = _cam([(200_000, True)], cur=150_000)
    assert c.plan(199_999, 0, 0) == (False, 150_000)                 # finished, but after t_end: the previous frame stays
    assert c.plan(200_000, 0, 0) == (True, 200_000)
    assert c.plan(None, 0, 0) == (True, 200_000)                      # no end yet: the newest finished frame
    c = _cam([(200_000, False)], cur=150_000)
    assert c.plan(250_000, 0, 0) == (False, 150_000)                  # not finished: the previous frame stays, the window grows
    first = _cam([(0, False)])
    assert first.plan(1_000, -49_000, 0) == (True, 0)                # the first frame is taken whatever its state
    # plan changes nothing; take applies its choice
    c = _cam([(200_000, True)], cur=150_000)
    take, cut = c.plan(210_000, 160_000, 0)
    assert c.cur_frame == (0, 150_000) and c.pending is not None
    c.take(take, cut)
    assert c.cur_frame == (1, 200_000) and c.pending is None and c.begin == 200_000


def test_steps_without_a_frame_at_or_before_t_end_are_refused():
    with pytest.raises(ValueError, match="first frame"):
        _cam([(5_000, True)]).plan(4_999, 0, 0)
    c = _cam(cur=300_000)                                             # frames set more than one frame ahead of the chunks
    with pytest.raises(ValueError, match="frame in use"):
        c.plan(250_000, 200_000, 0)


def test_window_cuts_refuse_before_any_camera_changes():
    from dagr_b200.streaming import _FusionDetector

    class Stub(_FusionDetector):
        since_frame = True

    det = Stub()
    det._cams = [_cam([(10_000, True)], cur=0), _cam([(20_000, True)])]
    with pytest.raises(ValueError, match="camera 0"):
        det._window_cuts([0, 0], [15_000, 15_000], [0, 0])           # camera 1's first frame is after t_end
    assert det._cams[0].cur_frame == (0, 0) and det._cams[0].pending is not None
    cuts = det._window_cuts([-35_000, -30_000], [15_000, 20_000], [0, 0])
    assert cuts == [10_000, 20_000] and [c.cur_frame[1] for c in det._cams] == [10_000, 20_000]
    det.since_frame = False                                           # the sliding window: the cuts as they come
    assert det._window_cuts([1, 2], [3, 4], [0, 0]) == [1, 2]


def test_frame_times_are_required_and_ordered_before_any_device_work():
    import torch
    c = _cam()
    img = torch.zeros((3, _Det.H, _Det.W), dtype=torch.uint8)
    with pytest.raises(ValueError, match="needs t_us"):
        c.set(img, None)
    c.last_t = 1_000
    with pytest.raises(ValueError, match="older than"):
        c.set(img, 999)
    assert c.nframes == 0 and c.pending is None
    assert c.check_time(1_000) == 1_000                               # equal times are in order


def test_since_frame_needs_an_image_fusion_model():
    from dagr_b200.streaming import FusionMultiStreamDetector, FusionStreamingDetector
    events_only, _ = make_model("n", 180, 240)
    with pytest.raises(ValueError, match="image-fusion"):
        FusionStreamingDetector(events_only, since_frame=True)
    with pytest.raises(ValueError, match="image-fusion"):
        FusionMultiStreamDetector(events_only, streams=2, since_frame=True)


def test_cut_stage_is_the_push_stage_at_max_chunk_one():
    from dagr_b200.streaming import CUT_STAGE, pack_cut_stage
    st = np.full(3 * CUT_STAGE + 5, -7, np.int32)
    pack_cut_stage(st, [100, -200, 2**31 - 1], planes=[1, 2, 5])
    assert st[:12].reshape(3, 4).tolist() == [[0, 100, 0, 1], [0, -200, 0, 2], [0, 2**31 - 1, 0, 5]]
    assert not st[12:24].any() and (st[24:] == -7).all()              # 4*S event words, zero; nothing past the block
    pack_cut_stage(st, [4, 5, 6])
    assert st[:12].reshape(3, 4)[:, 3].tolist() == [0, 0, 0]
    with pytest.raises(ValueError, match="smaller"):
        pack_cut_stage(np.zeros(CUT_STAGE * 2, np.int32), [1, 2, 3])


def test_chunk_stage_layouts_are_unchanged():
    from dagr_b200.streaming import pack_raw_stage, pack_stage
    c = (np.array([1, 2], np.int16), np.array([3, 4], np.int16), np.array([10, 11], np.int32), np.array([1, -1], np.int8))
    st = np.full(4 + 4 * 3, -7, np.int32)
    assert pack_stage(st, [c], [5], 3) == [2]
    assert st.tolist() == [2, 5, 0, 0, 1, 3, 10, 1, 2, 4, 11, -1, -7, -7, -7, -7]
    raw = np.full(4 + 2 * 3, -7, np.int32)
    assert pack_raw_stage(raw, [(c[0], c[1], c[2], np.array([1, 0], np.int8))], [5], 3) == [2]
    assert raw.tolist() == [2, 5, 0, 0, 1 | 3 << 16 | -(1 << 31), 10, 2 | 4 << 16, 11, -7, -7]


def test_two_pushes_leave_exactly_the_window_since_the_frame():
    """the host model of dagr_stream_push[_multi]: a chunk that straddles t_cut keeps its older rows after the first push;
    the cut stage pushed behind it removes them, and window_state's counts follow from the two control blocks."""
    from dagr_b200.streaming import CUT_STAGE, pack_cut_stage, pack_stage
    from tests.test_graph_sort_cpu import CTL, RingModel
    S, cap, mc = 2, 64, 8
    m = RingModel(S, cap, mc)
    cut1 = np.zeros(S * CUT_STAGE, np.int32)

    def step(chunks, t_cut):
        st = m.stage(np.zeros((S, 4)))
        pack_stage(st, chunks, t_cut, mc)
        m.push(st)
        mid = m.ctl.copy()
        pack_cut_stage(cut1, t_cut)
        m.mc = 1
        m.push(cut1)
        m.mc = mc
        return mid

    def ev(ts):
        ts = np.asarray(ts, np.int32)
        return (ts % 7).astype(np.int16), (ts % 5).astype(np.int16), ts, np.ones(len(ts), np.int8)

    step([ev([1, 2, 3, 4]), ev([10, 11])], [0, 0])
    mid = step([ev([5, 6, 7, 8]), ev([12, 13, 14])], [6, 12])          # stream 0: the frame at 6 falls inside the chunk
    _, pos, _ = m.windows()
    assert pos[:, 2].tolist() == [6, 7, 8, 12, 13, 14]
    fin = m.ctl
    for s, (evicted, appended) in enumerate([(4, 3), (2, 3)]):
        b, a = mid[CTL * s:CTL * (s + 1)], fin[CTL * s:CTL * (s + 1)]
        assert (int(b[2]), int(b[3]) - int(a[2])) == (evicted, appended), s
        assert int(a[1]) == [3, 3][s] and int(a[3]) == 0
    assert int(fin[CTL * S]) == 6 and int(fin[CTL * 1 + 6]) == 3      # the window offsets and the total follow the second push
