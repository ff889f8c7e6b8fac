"""The JPEG slot's sample stages (decode front end, K3 resampler, encode back end) as the resize and conversion legs chain them:
one slot reused by chains whose buffers grow and shrink, the host-encoder path of a JPEG resize, grey sources, resizes to the
source's own size and compress_to_size with a resize.  Bar: every output equals the oracle's, byte for byte."""
import numpy as np
import pytest

import png_resize_cases as cases
from pngutil import pil_pixels, pil_png, synth
from test_png_resize_gpu import decode_exact, oracle_of, want_rgba
from test_webp_gpu import FMT_JPEG, FMT_PNG, FMT_WEBP, _jpeg_rgb, planar
from test_webp_lossless_gpu import _decoded_rgba, _soft_alpha, _webp
from webputil import pil_decode

pytestmark = pytest.mark.gpu


def _jpeg_params(L, w=0, q=85):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.width = q, 420, 1, w
    return p


def _resized(O, planes, nw, nh):
    return np.stack([O.resize_plane(np.ascontiguousarray(p), nw, nh) for p in planes])


def test_one_slot_reused_by_chains_that_grow_and_shrink(L, O, golden):
    """On one thread every call takes the same slot: a chain must not lose its planes to a buffer a later stage grows, and a
    small chain after a large one must not read stale layout."""
    from oracle import vp8l
    from tools.synth import synth_jpeg
    big = synth_jpeg(6000, 4000, 3)
    big_want = O.jpeg_lossy_resized(big, O.params(85, 420, True), 1920, 0)
    tiny = golden("in_420_tiny_17x9.jpg")
    tiny_want = O.webp_encode(_jpeg_rgb(O, tiny, *O.compute_dimensions(17, 9, 40, 0)), 75)[0]
    png = cases.make(O, 6, 16, False, 300, 200, seed=3)
    png_info, png_rows = oracle_of(O, png, 130, 0)
    h, w = 150, 210
    rgba = np.concatenate([synth(h, w, 3, seed=2, kind="photo"), _soft_alpha(h, w, 1)[:, :, None]], axis=2)
    webp = _webp(rgba, lossless=True, exact=True)
    px = _decoded_rgba(L, webp)
    nw, nh = O.compute_dimensions(w, h, 100, 0)
    webp_want = vp8l.webp_lossless_encode(np.ascontiguousarray(np.moveaxis(_resized(O, np.moveaxis(px, -1, 0), nw, nh), 0, -1)))
    vga = golden("in_420_base_640x480.jpg")
    lay, co = L.jpeg_decode_coefficients(vga)

    assert L.set_png_resize(True) == 0
    try:
        assert L.compress_in_memory(big, _jpeg_params(L, 1920)) == big_want
        p = L.default_params(); p.webp_quality = 75; p.width = 40
        assert L.convert_in_memory(tiny, p, FMT_WEBP) == tiny_want
        p = L.default_params(); p.png_optimize, p.png_optimization_level, p.width = 1, 3, 130
        got, _ = decode_exact(O, L.compress_in_memory(png["png"], p))
        assert np.array_equal(got, want_rgba(png_info, png_rows))
        p = L.default_params(); p.webp_lossless, p.width = 1, 100
        assert L.compress_in_memory(webp, p) == webp_want
        assert np.array_equal(L.jpeg_decode_planes(lay, co), O.Jpeg(vga).decode_native())
        assert L.compress_in_memory(big, _jpeg_params(L, 1920)) == big_want
    finally:
        L.set_png_resize(False)


@pytest.mark.parametrize("width", [200, 640])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_jpeg_resize_in_every_entropy_mode(L, O, golden, mode, width):
    """Modes 0 and 2 code the resized coefficients on the host, after they come back from the device."""
    data = golden("in_420_base_640x480.jpg")
    want = O.jpeg_lossy_resized(data, O.params(85, 420, True), width, 0)
    L.set_entropy_mode(mode)
    try:
        assert L.compress_in_memory(data, _jpeg_params(L, width)) == want
    finally:
        L.set_entropy_mode(3)


def test_grey_sources_with_resize(L, O, golden):
    """A grey source is one plane through the stages; only the WebP encoder sees it three times.  (Grey JPEG -> PNG with a resize
    is a parameter of test_webp_gpu.)"""
    data = golden("in_gray_base_355x237.jpg")
    nw, nh = O.compute_dimensions(355, 237, 120, 0)
    p = L.default_params(); p.webp_quality = 70; p.width = 120
    assert L.convert_in_memory(data, p, FMT_WEBP) == O.webp_encode(_jpeg_rgb(O, data, nw, nh), 70)[0]
    grey = synth(50, 70, 1, seed=5)
    op = O.params(80, 420, True)
    nw, nh = O.compute_dimensions(70, 50, 33, 0)
    assert L.convert_in_memory(pil_png(grey), _jpeg_params(L, 33, 80), FMT_JPEG) == O.write(O.forward(_resized(O, planar(grey), nw, nh), op), op)


def test_resize_to_the_source_size(L, O, golden):
    """The resampler enqueues nothing at the same size and the next stage reads the input planes.  (JPEG -> JPEG, JPEG -> WebP and
    PNG -> PNG at the source's size are parameters of test_resize_gpu, test_webp_gpu and test_png_resize_gpu.)"""
    data = golden("in_420_base_355x237.jpg")
    p = L.default_params(); p.png_optimize = 1; p.width = 355
    got = np.asarray(pil_pixels(L.convert_in_memory(data, p, FMT_PNG)).convert("RGB")).transpose(2, 0, 1)
    assert np.array_equal(got, _jpeg_rgb(O, data))
    rgb = synth(90, 120, 3, seed=4)
    p = L.default_params(); p.webp_quality = 80; p.width = 120
    assert L.convert_in_memory(pil_png(rgb), p, FMT_WEBP) == O.webp_encode(planar(rgb), 80)[0]
    op = O.params(80, 420, True)
    assert L.convert_in_memory(pil_png(rgb), _jpeg_params(L, 120, 80), FMT_JPEG) == O.write(O.forward(O.rgb_to_ycc(planar(rgb)), op), op)
    src = _webp(rgb, quality=90)
    p = L.default_params(); p.png_optimize = 1; p.height = 90
    got = np.asarray(pil_pixels(L.convert_in_memory(src, p, FMT_PNG)).convert("RGB"))
    assert np.array_equal(got, pil_decode(src))


def test_webp_compress_to_size_with_resize(L, O):
    """The resized planes stay on the slot for every quality the bisection tries."""
    src = _webp(synth(240, 320, 3, seed=9, kind="photo"), quality=90)
    nw, nh = O.compute_dimensions(320, 240, 150, 0)
    rz = _resized(O, planar(pil_decode(src)), nw, nh)
    target = len(O.webp_encode(rz, 80)[0]) * 3 // 4
    p = L.default_params(); p.webp_quality = 80; p.width = 150
    out = L.compress_to_size_in_memory(src, p, target)
    assert len(out) <= target
    assert out == O.webp_encode(rz, int(p.webp_quality))[0]
