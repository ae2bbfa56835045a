"""PipelinedDetector with image fusion without a GPU: the refusal of --no_events models and the argument checks of
submit(), which all run before any device work (on CPU inputs a forward would fail with RuntimeError instead, and the
engine would count launches)."""
import pytest
import torch

from dagr_b200.data import format_data, synth_batch
from tests.helpers import make_model

W, H, B = 240, 180, 2


def _data(**image):
    d = format_data(synth_batch(B, 500, W, H, seed=3, with_image=True))
    for k, v in image.items():
        setattr(d, k, v)
    return d


def _refused(model, data, match):
    from dagr_b200.pipeline import PipelinedDetector
    pd = PipelinedDetector(model)
    with pytest.raises(ValueError, match=match):
        pd.submit(data)
    assert model.engine.launches == 0 and model.engine.overlap is False
    assert model._image_branch is None, "the image branch was reached"


def test_no_events_model_is_refused():
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18", no_events=True)
    _refused(model, _data(), "no_events")


@pytest.mark.parametrize("case", ["missing", "not_a_tensor", "three_dims", "four_channels", "int32", "batch", "device"])
def test_submit_checks_the_frames_before_device_work(case):
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18")
    img = torch.rand(B, 3, H, W)
    bad = dict(missing=None, not_a_tensor=img.numpy(), three_dims=img[0], four_channels=torch.rand(B, 4, H, W),
               int32=(img * 255).int(), batch=torch.rand(B + 1, 3, H, W), device=torch.empty(B, 3, H, W, device="meta"))[case]
    match = dict(missing="needs data.image", not_a_tensor="needs data.image", batch="frames for a batch of",
                 device="data.image is on").get(case, "expected u8 or float frames")
    _refused(model, _data(image=bad), match)


def test_keep_stream_is_refused():
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18")
    model.keep_stream = True
    _refused(model, _data(image=torch.rand(B, 3, H, W)), "keep_stream")


def test_u8_and_float_frames_pass_the_checks():
    from dagr_b200.pipeline import PipelinedDetector
    model, _ = make_model("n", H, W, use_image=True, img_net="resnet18")
    pd = PipelinedDetector(model)
    for img in (torch.randint(0, 256, (B, 3, H, W), dtype=torch.uint8), torch.rand(B, 3, H, W)):
        pd._check(_data(image=img))
