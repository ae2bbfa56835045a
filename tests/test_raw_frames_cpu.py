"""Raw camera frames without a GPU: the integer restatement of the reference's frame preparation (dsec_data.py:149-154)
against the golden vectors its unmodified method produced, and against OpenCV itself where it is installed; the argument
contract of dagr_frame_preprocess (every bad input is refused with DAGR_E_ARG and a message before anything is launched);
and the constructor checks of raw_frames on the fusion detectors."""
import ctypes as C
from pathlib import Path

import numpy as np
import pytest

from tests.helpers import make_model

E_ARG = -1
BAD = C.c_void_p(256)          # never dereferenced: every call below fails its argument check first
GOLD_PATH = Path(__file__).resolve().parent / "golden" / "frame_golden.npz"


def test_frame_oracle_equals_reference_golden():
    from oracle.ref_frame import preprocess_image
    g = np.load(GOLD_PATH)
    assert int(g["cases"]) == 7
    for i in range(int(g["cases"])):
        h, w, s = (int(v) for v in g[f"c{i}_geom"])
        img, want = g[f"c{i}_in"], g[f"c{i}_out"]
        assert want.shape == (1, 3, h, w) and want.dtype == np.uint8
        assert np.array_equal(preprocess_image(img, h, w, s), want), i
    assert {int(g[f"c{i}_geom"][2]) for i in range(7)} == {1, 2, 3, 4}
    assert any(g[f"c{i}_in"].shape[0] > g[f"c{i}_geom"][0] * g[f"c{i}_geom"][2] for i in range(7))     # a cropped case


def test_frame_oracle_equals_opencv_on_random_frames():
    cv2 = pytest.importorskip("cv2")
    from oracle.ref_frame import preprocess_image
    rng = np.random.default_rng(21)
    for i in range(50):
        s = 1 + i % 5
        h, w = int(rng.integers(2, 30)), int(rng.integers(2, 40))
        img = rng.integers(0, 256, (s * h + int(rng.integers(0, 5)), s * w, 3), dtype=np.uint8)
        if i % 3 == 1:
            img = (img > 127).astype(np.uint8) * 255                   # saturating edges
        want = cv2.resize(img[:s * h], (w, h), interpolation=cv2.INTER_CUBIC).transpose(2, 0, 1)[None]
        assert np.array_equal(preprocess_image(img, h, w, s), want), (i, s, h, w)


def test_frame_oracle_rounds_half_to_even():
    """a 2x2 crop with rows (v, 0) down-sized to one pixel: the clamped vertical taps read rows 0, 0, 1, 1, so the sum is
    (-3 + 19) * v * 32 = 512 v and the output v / 2 -- a tie for odd v, which OpenCV rounds to even."""
    from oracle.ref_frame import resize_int
    for v, want in ((1, 0), (3, 2), (5, 2), (4, 2), (255, 128), (253, 126)):
        crop = np.zeros((2, 2, 1), np.uint8)
        crop[0, :] = v
        assert resize_int(crop, 1, 1, 2)[0, 0, 0] == want, v


def _fp(lib, frames=BAD, n=1, sh=480, sw=640, s=2, h=215, w=320, out_u8=BAD, out_f32=None, lut=None):
    return lib.dagr_frame_preprocess(frames, n, sh, sw, s, h, w, out_u8, out_f32, lut, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(frames=None), "null frames"),
    (dict(out_u8=None), "exactly one"),
    (dict(out_f32=BAD), "exactly one"),
    (dict(out_u8=None, out_f32=BAD), "lut"),
    (dict(n=0), "nframes"),
    (dict(n=65536), "nframes"),
    (dict(w=0), "out_w"),
    (dict(h=0), "out_h"),
    (dict(s=0), "scale"),
    (dict(sw=641), "src_w"),
    (dict(s=3), "src_w"),
    (dict(sh=429), "src_h"),
])
def test_frame_preprocess_rejects_bad_arguments(kw, needle):
    from dagr_b200 import _lib
    lib = _lib.load()
    assert _fp(lib, **kw) == E_ARG
    msg = lib.dagr_last_error().decode()
    assert "dagr_frame_preprocess" in msg and needle in msg, msg


def test_raw_frames_needs_a_sensor_and_an_integer_scale():
    from dagr_b200.streaming import FusionMultiStreamDetector, FusionStreamingDetector
    model, _ = make_model("n", 215, 320, use_image=True, img_net="resnet18")
    for kw, needle in [(dict(raw_frames=True), "sensor"), (dict(raw_frames=True, sensor=(641, 480)), "integer multiple"),
                       (dict(raw_frames=True, sensor=(640, 429)), "integer multiple")]:
        with pytest.raises(ValueError, match=needle):
            FusionStreamingDetector(model, **kw)
        with pytest.raises(ValueError, match=needle):
            FusionMultiStreamDetector(model, streams=2, **kw)
    with pytest.raises(RuntimeError, match="CUDA"):                   # a valid sensor gets as far as the device check
        FusionStreamingDetector(model, sensor=(640, 480), raw_frames=True)


def test_preprocess_image_needs_cuda_frames():
    import torch
    from dagr_b200 import ingest
    with pytest.raises(RuntimeError, match="CUDA"):
        ingest.preprocess_image(torch.zeros((480, 640, 3), dtype=torch.uint8), 215, 320, 2)
