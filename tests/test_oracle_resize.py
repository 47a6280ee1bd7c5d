"""The numpy integer restatements in oracle/resize.py must be bit-exact against the libraries the
reference's callers use (Pillow for Models/visualizations, OpenCV for the C++ backends)."""
import numpy as np
import pytest

from oracle import resize, synth


@pytest.mark.parametrize("kind", ["natural", "iid"])
def test_pil_bicubic_1080p(kind):
    from PIL import Image
    f = synth.synth_frame(7, kind=kind)
    got = resize.pil_bicubic_resize(f, 640, 320)
    exp = np.asarray(Image.fromarray(f).resize((640, 320)))   # default filter == BICUBIC
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("kind", ["natural", "iid"])
def test_cv_linear_1080p_and_egolanes_crop(kind):
    import cv2
    f = synth.synth_frame(9, kind=kind)
    assert np.array_equal(resize.cv_linear_resize(f, 640, 320), cv2.resize(f, (640, 320)))
    crop = np.ascontiguousarray(f[420:])                       # main.cpp:497-502
    assert np.array_equal(resize.cv_linear_resize(crop, 640, 320),
                          cv2.resize(crop, (640, 320), interpolation=cv2.INTER_LINEAR))


@pytest.mark.parametrize("h,w", [(700, 401), (333, 517), (320, 640), (480, 640), (2160, 3840)])
def test_ragged_sizes(h, w):
    import cv2
    from PIL import Image
    rng = np.random.default_rng(h * 7 + w)
    f = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    assert np.array_equal(resize.pil_bicubic_resize(f, 640, 320),
                          np.asarray(Image.fromarray(f).resize((640, 320))))
    assert np.array_equal(resize.cv_linear_resize(f, 640, 320), cv2.resize(f, (640, 320)))


@pytest.mark.parametrize("h,w,oh,ow", [
    (1080, 1920, 512, 910),      # downscale: the 1080p letterbox
    (333, 517, 320, 640),        # one axis down, one up
    (100, 130, 256, 333),        # upscale
    (5, 8, 320, 640),            # upscale from a few pixels
    (270, 480, 270, 480),        # identity
    (1, 4800, 1, 640),           # 1-pixel axis kept, the other down
    (1, 1, 320, 640),            # a 1x1 frame
    (7, 1, 512, 3),              # a 1-pixel column
    (2400, 4800, 320, 640),      # a 7.5x downscale (17 taps)
])
def test_pil_bilinear_matches_pillow(h, w, oh, ow):
    from PIL import Image
    rng = np.random.default_rng(h * 31 + w)
    f = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    exp = np.asarray(Image.fromarray(f).resize((ow, oh), Image.BILINEAR))
    assert np.array_equal(resize.pil_bilinear_resize(f, ow, oh), exp)


def test_identity_size_is_passthrough():
    f = synth.synth_frame(1, 320, 640)
    assert np.array_equal(resize.pil_bicubic_resize(f, 640, 320), f)


def test_frames_are_deterministic():
    a, b = synth.synth_frame(5, 90, 160), synth.synth_frame(5, 90, 160)
    assert np.array_equal(a, b) and a.dtype == np.uint8 and a.shape == (90, 160, 3)
    assert not np.array_equal(a, synth.synth_frame(6, 90, 160))
    assert synth.stream_seed(3, 17) == 3017
