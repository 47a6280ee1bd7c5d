"""The device JPEG decoder (vpb_jpeg_decode) on hand-built streams, against cv2.imdecode byte for byte in both channel
orders: the matrix of tests/test_jpeg_streams_cpu.py (custom Huffman tables in every slot, slow self-synchronisation on
1, 2 and 67 CTAs, every partition and restart edge of the Huffman kernel, every coefficient category at its extremes,
every geometry residue), mixed-size batches, one decoder through growing and shrinking calls, and outputs inside
sentinel margins that must stay untouched.

The coefficients stay inside the decoder's contract: dequantised values of at most 4x an 8-bit image's range and
samples within the range limit's [-512, 511].  Past that, libjpeg-turbo's SIMD IDCT (cv2's CPU path) saturates and
overflows where jidctint.c wraps, and cv2's own result depends on its CPU."""
import numpy as np
import pytest
import torch

from autoware_vision_pilot_b200 import _lib as L
from tests.test_jpeg_cpu import encode, imdecode, natural
from tests.test_jpeg_streams_cpu import matrix

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

MARGIN = 4096                                            # sentinel bytes before and after every output
SENTINEL = 0xA5


def _decode(dec, streams, bgr):
    """decode into outputs inside larger buffers; the outputs, and a check that the margins are untouched"""
    objs = [L.JPEG(b) for b in streams]
    bufs = [torch.full((2 * MARGIN + o.h * o.w * 3,), SENTINEL, dtype=torch.uint8, device="cuda") for o in objs]
    dec.decode(objs, [b.data_ptr() + MARGIN for b in bufs], bgr)
    torch.cuda.synchronize()
    out = []
    for o, b in zip(objs, bufs):
        h = b.cpu().numpy()
        assert (h[:MARGIN] == SENTINEL).all() and (h[MARGIN + o.h * o.w * 3:] == SENTINEL).all(), "margin written"
        out.append(h[MARGIN:MARGIN + o.h * o.w * 3].reshape(o.h, o.w, 3))
    return out


def _check(got, streams, bgr, what):
    for g, b in zip(got, streams):
        exp = imdecode(b)
        assert np.array_equal(g, exp if bgr else exp[:, :, ::-1]), (what, bgr)


@pytest.fixture(scope="module")
def dec():
    d = L.JpegDecoder(2400, 4800, 8)
    yield d
    d.close()


@pytest.mark.parametrize("bgr", [True, False])
def test_matrix_one_stream_per_call(dec, bgr):
    for label, b in matrix():
        _check(_decode(dec, [b], bgr), [b], bgr, label)


def test_matrix_in_mixed_batches_of_8(dec):
    m = matrix()
    order = np.random.default_rng(0).permutation(len(m))
    for k in range(0, len(order) - 7, 8):
        chunk = [m[i] for i in order[k:k + 8]]
        bgr = k % 16 == 0
        _check(_decode(dec, [b for _, b in chunk], bgr), [b for _, b in chunk], bgr, [label for label, _ in chunk])


def test_decoder_state_through_growth_and_shrinking():
    """one decoder: small streams, the largest frame it takes (4800x2400 random q100 4:4:4, thousands of CTAs, the
    staging and the CTA chains grow), small streams again, then calls whose CTA counts keep changing.  The oracle is
    pinned to cv2 on a 240x480 stream of the same kind ("random q100" of the matrix); this one is checked against cv2
    directly."""
    big = encode(np.random.default_rng(9).integers(0, 256, (2400, 4800, 3), dtype=np.uint8), 100, "444")
    m = matrix()
    small = [b for label, b in m if label.startswith(("geometry", "single", "under"))][:8]
    slow = [b for label, b in m if label.startswith("slow-sync")]
    d = L.JpegDecoder(2400, 4800, 8)
    _check(_decode(d, small, True), small, True, "small before")
    _check(_decode(d, [big], True), [big], True, "4800x2400")
    _check(_decode(d, small, False), small, False, "small after")
    for b in (slow[2], small[0], big, slow[0], slow[1], small[1], slow[5], big, small[2]):
        _check(_decode(d, [b], True), [b], True, "changing CTA counts")
    _check(_decode(d, [big, small[3], slow[2], small[4]], True), [big, small[3], slow[2], small[4]], True, "batch")
    d.close()

