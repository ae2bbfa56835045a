"""CPU restatement of the reference's camera-frame preparation (TEST INFRASTRUCTURE ONLY -- never imported by the product
path): src/dagr/data/dsec_data.py:149-154, `DSEC.preprocess_image`.

    image = image[:scale * height]                                                     # crop rows
    image = cv2.resize(image, (width, height), interpolation=cv2.INTER_CUBIC)          # integer factor `scale`
    image = torch.from_numpy(image).permute(2, 0, 1).unsqueeze(0)                      # HWC -> [1, 3, H, W] u8

The reference only resizes by an integer factor: the crop makes the height `scale * height`, and the sensor width is
`scale * width`.  At an integer factor OpenCV's INTER_CUBIC on uint8 is integer arithmetic, restated here:
  * separable cubic with A = -0.75, taps at source offsets -1..+2, source indices clamped to the cropped image
    (replicated border);
  * the source coordinate of output pixel d is (d + 0.5) * scale - 0.5.  Even scale: sx = scale * d + scale / 2 - 1,
    fraction 0.5, taps sx - 1 .. sx + 2 with weights [-3, 19, 19, -3] / 32 (the cubic at 0.5, exact in binary).  Odd
    scale: the fraction is 0 and output pixel d is source pixel `scale * d + (scale - 1) / 2`;
  * the sum of wy * wx * src in integers (units of 1/1024), rounded half to even, saturated to [0, 255].
Half-up rounding ((v + 512) >> 10) does not reproduce OpenCV; half to even does (tests/test_raw_frames_cpu.py checks
this against cv2.resize where OpenCV is installed).  Pinned by tests/golden/frame_golden.npz, generated from the
reference's unmodified method (tests/golden/make_frame_golden.py).
"""
import numpy as np

CUBIC_HALF = np.array([-3, 19, 19, -3], dtype=np.int64)          # cubic weights at fraction 0.5, in units of 1/32


def resize_int(crop, height, width, scale):
    """crop u8 [scale*height, scale*width, C] -> u8 [height, width, C]: cv2.resize(INTER_CUBIC) at integer factor `scale`."""
    s = int(scale)
    src = np.asarray(crop).astype(np.int64)
    if s % 2 == 1:
        o = (s - 1) // 2
        return src[o::s][:height, o::s][:, :width].astype(np.uint8)
    sx = lambda n: s * np.arange(n) + s // 2 - 1                                     # floor((d + 0.5) * s - 0.5)
    iy = np.clip(sx(height)[:, None] + np.arange(-1, 3), 0, src.shape[0] - 1)        # [H, 4] clamped rows
    ix = np.clip(sx(width)[:, None] + np.arange(-1, 3), 0, src.shape[1] - 1)         # [W, 4] clamped columns
    v = np.zeros((height, width, src.shape[2]), dtype=np.int64)
    for ky in range(4):
        for kx in range(4):
            v += CUBIC_HALF[ky] * CUBIC_HALF[kx] * src[iy[:, ky]][:, ix[:, kx]]
    q, r = v >> 10, v & 1023                                                         # floor(v / 1024), remainder
    q += (r > 512) | ((r == 512) & (q & 1 == 1))                                     # round half to even
    return np.clip(q, 0, 255).astype(np.uint8)


def preprocess_image(image, height, width, scale):
    """dsec_data.py:149-154: u8 [sh, sw, 3] (sh >= scale*height, sw == scale*width, channel order passed through) ->
    u8 [1, 3, height, width]."""
    image = np.asarray(image)
    sh, sw = image.shape[:2]
    if scale < 1 or sw != scale * width or sh < scale * height:
        raise ValueError(f"frame {sw}x{sh} is not an integer multiple {scale} of {width}x{height}")
    out = resize_int(image[:scale * height], height, width, scale)
    return np.ascontiguousarray(out.transpose(2, 0, 1))[None]
