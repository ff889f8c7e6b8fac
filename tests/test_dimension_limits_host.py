"""JPEG's dimension limit on the host side of every entry point that parses a JPEG.

libjpeg-turbo and mozjpeg refuse a side over JPEG_MAX_DIMENSION = 65500 although the SOF field holds up to 65535.  The header
is read before any device is needed, so a source over the limit is corrupt input (code 4) on every entry point, with or without
a GPU: the lossless transcode, which falls back to the host transcoder without a device, must refuse it as well instead of
writing a file no libjpeg-based decoder opens.  The limit is pinned to Pillow's libjpeg-turbo, not to a number written here."""
import io

import numpy as np
import pytest
from PIL import Image

LIMIT = 65500
ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
               35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


def _image(w, h, grey, seed=0):
    rng = np.random.default_rng(seed)
    ramp = np.add.outer(np.arange(h), np.arange(w))
    if grey:
        return ((ramp % 256) ^ rng.integers(0, 16, (h, w))).astype(np.uint8)
    return ((ramp[..., None] * np.array([1, 3, 7]) % 256) ^ rng.integers(0, 16, (h, w, 3))).astype(np.uint8)


def jpeg_at(w, h, grey, progressive=False):
    """a Pillow (libjpeg-turbo) JPEG of w x h: 4:2:0 YCbCr or one grey component"""
    b = io.BytesIO()
    Image.fromarray(_image(w, h, grey)).save(b, "JPEG", quality=90, subsampling=2, progressive=progressive)
    return b.getvalue()


def patch_sof(data, w=None, h=None):
    """the same file with its frame header's width and / or height rewritten"""
    d, i = bytearray(data), 2
    while i + 4 <= len(d):
        assert d[i] == 0xFF
        m, n = d[i + 1], d[i + 2] << 8 | d[i + 3]
        if m in (0xC0, 0xC1, 0xC2):
            if h is not None:
                d[i + 5:i + 7] = h.to_bytes(2, "big")
            if w is not None:
                d[i + 7:i + 9] = w.to_bytes(2, "big")
            return bytes(d)
        i += 2 + n
    raise AssertionError("no SOF")


# (name, grey, wide): wide = the long side is the width (LIMIT x 8), else the height (8 x LIMIT)
VARIANTS = [("420_wide", False, True), ("420_tall", False, False), ("grey_wide", True, True), ("grey_tall", True, False)]
_cache = {}


def at_limit(grey, wide):
    key = (grey, wide)
    if key not in _cache:
        _cache[key] = jpeg_at(LIMIT, 8, grey) if wide else jpeg_at(8, LIMIT, grey)
    return _cache[key]


def over(grey, wide, side):
    return patch_sof(at_limit(grey, wide), w=side) if wide else patch_sof(at_limit(grey, wide), h=side)


def test_pillow_pins_the_limit():
    """libjpeg-turbo writes and reads LIMIT, and refuses LIMIT + 1 both ways"""
    for grey, wide in ((False, True), (True, False)):
        data = at_limit(grey, wide)
        im = Image.open(io.BytesIO(data))
        im.load()
        assert im.size == ((LIMIT, 8) if wide else (8, LIMIT))
        bad = over(grey, wide, LIMIT + 1)
        with pytest.raises(OSError):
            Image.open(io.BytesIO(bad)).load()
    for size in ((LIMIT + 1, 8), (8, LIMIT + 1)):
        with pytest.raises(OSError):
            Image.new("RGB", size).save(io.BytesIO(), "JPEG")


def _code(L, call):
    with pytest.raises(L.B200Error) as e:
        call()
    return e.value.code, str(e.value)


@pytest.mark.parametrize("side", [LIMIT + 1, 65535])
@pytest.mark.parametrize("name,grey,wide", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_sources_over_the_limit_are_corrupt_input(L, name, grey, wide, side):
    data = over(grey, wide, side)
    p = L.default_params()
    png = L.default_params()
    png.png_optimize = 1
    lossless = L.default_params()
    lossless.jpeg_optimize = 1
    calls = {
        "compress": lambda: L.compress_in_memory(data, p),
        "lossless transcode": lambda: L.compress_in_memory(data, lossless),
        "resize": lambda: L.compress_in_memory(data, _resize(L, 100)),
        "to png": lambda: L.convert_in_memory(data, png, L.FMT_PNG),
        "to webp": lambda: L.convert_in_memory(data, p, L.FMT_WEBP),
        "to size": lambda: L.compress_to_size_in_memory(data, L.default_params(), 5000),
        "coefficients": lambda: L.jpeg_decode_coefficients(data),
    }
    for what, call in calls.items():
        code, msg = _code(L, call)
        assert code == L.ERR_CORRUPT_INPUT, (what, code, msg)
        assert "Maximum supported image dimension is 65500 pixels" in msg, (what, msg)
    (out, code, msg), = L.compress_batch([data], lossless, n_threads=1)
    assert out is None and code == L.ERR_CORRUPT_INPUT, msg


@pytest.mark.parametrize("name,grey,wide", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_lossless_transcode_over_the_limit_writes_nothing(L, name, grey, wide):
    """without a device this leg is the host transcoder, which needs no device to turn a 65501-wide source into a file that
    libjpeg-turbo cannot open: the header refusal must come first"""
    p = L.default_params()
    p.jpeg_optimize = 1
    code, msg = _code(L, lambda: L.compress_in_memory(over(grey, wide, LIMIT + 1), p))
    assert code == L.ERR_CORRUPT_INPUT, msg


def _resize(L, width):
    p = L.default_params()
    p.width = width
    return p


@pytest.mark.parametrize("side", [LIMIT + 1, 65535])
@pytest.mark.parametrize("name,grey,wide", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_the_oracle_refuses_the_same_files(O, name, grey, wide, side):
    data = over(grey, wide, side)
    for call in (lambda: O.Jpeg(data), lambda: O.jpeg_lossy(data, O.params(80, 420, True)), lambda: O.jpeg_lossless(data, O.params(80, 420, True)),
                 lambda: O.jpeg_lossy_resized(data, O.params(80, 420, True), 100, 0)):
        with pytest.raises(O.OracleError, match="Maximum supported image dimension is 65500 pixels"):
            call()


@pytest.mark.parametrize("progressive", [False, True])
@pytest.mark.parametrize("name,grey,wide", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_sources_at_the_limit_are_read(L, O, name, grey, wide, progressive):
    """LIMIT itself is a legal JPEG: its coefficients are the oracle's, and the lossless transcode (on the device when there is
    one, else the host transcoder) is the oracle's file, which libjpeg-turbo decodes to the source's pixels"""
    data = at_limit(grey, wide) if not progressive else jpeg_at(*((LIMIT, 8) if wide else (8, LIMIT)), grey, progressive=True)
    lay, coefs = L.jpeg_decode_coefficients(data)
    assert (lay.width, lay.height) == ((LIMIT, 8) if wide else (8, LIMIT))
    ref = O.Jpeg(data)
    for c in range(lay.ncomp):
        assert np.array_equal(L.component_view(lay, coefs, c), ref.coef(c)[:, :, ZZ])
    p = L.default_params()
    p.jpeg_optimize = 1
    out = L.compress_in_memory(data, p)
    assert out == O.jpeg_lossless(data, O.params(80, 0, True))
    src = np.asarray(Image.open(io.BytesIO(data)))
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(out))), src)


def test_target_limit_in_the_oracle(O):
    """the twin of a resize to JPEG refuses a target side over LIMIT and accepts LIMIT"""
    small = jpeg_at(40, 8, False)
    with pytest.raises(O.OracleError, match="invalid target dimensions"):
        O.jpeg_lossy_resized(small, O.params(80, 420, True), LIMIT + 1, 8)
    out = O.jpeg_lossy_resized(small, O.params(80, 420, True), LIMIT, 8)
    im = Image.open(io.BytesIO(out))
    im.load()
    assert im.size == (LIMIT, 8)
    with pytest.raises(O.OracleError, match="invalid target dimensions"):
        O.forward(np.zeros((1, 8, LIMIT + 1), np.uint8), O.params(80, 0, False))
