"""The lossless WebP palette switch on the device (b200_set_webp_palette): with it on, every lossless WebP leg -- `--lossless` on
WebP sources, PNG and JPEG -> lossless WebP, the lossless frames of animated WebP -- writes the palette twin's file
(oracle/vp8l_palette_oracle.c) byte for byte, libwebp decodes it to exactly the coded pixels, a file is never larger than with the
switch off, and images of more than 256 colours keep today's bytes.  Every fixture that turns a switch on turns it off again."""
import io
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import webp_anim_cases as wc
from png_webp_cases import cases, expected_rgba, make_case
from pngutil import pil_png, synth
from webp_palette_cases import coloured, sprite_sheet, two_colour_bitmap

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def OV(O):
    from oracle import vp8l
    return vp8l


@pytest.fixture(scope="module")
def OP(O):
    from oracle import vp8l_palette
    return vp8l_palette


@pytest.fixture
def pal(L):
    assert L.lib().b200_init_device(0) == 0
    assert L.set_webp_palette(1) == 0
    try:
        yield L
    finally:
        L.set_webp_palette(0)


@pytest.fixture
def convert(pal):
    assert pal.set_webp_lossless_convert(1) == 0
    try:
        yield pal
    finally:
        pal.set_webp_lossless_convert(0)


def _params(L, **kw):
    p = L.default_params(); p.webp_lossless = 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _webp(img, **kw):
    from PIL import Image
    b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", **kw)
    return b.getvalue()


def _pil_rgba(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data)); im.load()
    return np.asarray(im.convert("RGBA"))


def _decoded_rgba(L, data):
    rgb, a = L.webp_decode_rgba(data)
    if a is None:
        a = np.full(rgb.shape[:2], 255, np.uint8)
    return np.ascontiguousarray(np.concatenate([rgb, a[:, :, None]], axis=2))


def _check(out, OP, rgba):
    assert out == OP.webp_palette_encode(rgba)
    assert np.array_equal(_pil_rgba(out), rgba)


def _sample(name):
    with open(os.path.join(ROOT, "tests", "golden", "reference_samples", name), "rb") as f:
        return f.read()


def _webp_sources():
    yield "w0", _sample("w0.webp")
    yield "w1", _sample("w1.webp")
    yield "flat", _webp(synth(97, 131, 3, seed=5, kind="flat"), lossless=True)
    yield "flat_alpha_hidden", _webp(coloured(61, 83, 40, seed=3, alpha="hidden"), lossless=True, exact=True)
    yield "translucent_5", _webp(coloured(33, 77, 5, seed=4, alpha="translucent"), lossless=True, exact=True)
    yield "bitmap_odd_width", _webp(two_colour_bitmap(45, 203), lossless=True)
    yield "sprite", _webp(sprite_sheet(96, 144), lossless=True, exact=True)
    yield "one_pixel", _webp(np.array([[[9, 8, 7]]], np.uint8), lossless=True)
    yield "one_column", _webp(coloured(300, 1, 3, seed=6), lossless=True)
    yield "lossy_photo", _webp(synth(150, 210, 3, seed=12, kind="photo"), quality=80)


@pytest.mark.parametrize("case", list(_webp_sources()), ids=lambda c: c[0])
def test_webp_sources_match_the_twin(pal, OP, OV, case):
    _, src = case
    px = _decoded_rgba(pal, src)
    out = pal.compress_in_memory(src, _params(pal))
    _check(out, OP, px)
    assert len(out) <= len(OV.webp_lossless_encode(px))


PNG_CASES = [c for c in cases() if c[3] in (0, 3)]          # grey and palette PNGs at every depth, with and without tRNS


@pytest.mark.parametrize("case", PNG_CASES, ids=lambda c: c[0])
def test_palette_and_grey_pngs_match_the_twin(convert, O, OP, case):
    L = convert
    _, w, h, ct, bd, trns, plte_len = case
    data, raw, plte, t = make_case(w, h, ct, bd, seed=w * 31 + h * 7 + ct * 5 + bd, trns=trns, plte_len=plte_len)
    info, rows = L.png_decode(data)
    rgba = np.ascontiguousarray(expected_rgba(rows, info.width, info.color_type, info.bit_depth, plte, t))
    _check(L.convert_in_memory(data, _params(L), L.FMT_WEBP), OP, rgba)


def test_pillow_palette_png(convert, OP):
    from PIL import Image
    data = pil_png(Image.fromarray(synth(123, 301, 3, seed=9, kind="flat")).quantize(17))
    _check(convert.convert_in_memory(data, _params(convert), convert.FMT_WEBP), OP, _pil_rgba(data))


@pytest.mark.parametrize("name", ["in_gray_base_355x237.jpg", "in_420_base_355x237.jpg"])
def test_jpeg_matches_the_twin(convert, O, OP, OV, golden, name):
    data = golden(name)
    ycc = O.Jpeg(data).decode_native()
    rgb = O.ycc_to_rgb(ycc) if ycc.shape[0] == 3 else np.repeat(ycc, 3, axis=0)
    rgba = np.ascontiguousarray(np.concatenate([rgb.transpose(1, 2, 0), np.full(rgb.shape[1:] + (1,), 255, np.uint8)], axis=2))
    out = convert.convert_in_memory(data, _params(convert), convert.FMT_WEBP)
    _check(out, OP, rgba)
    st = OP.webp_palette_stages(rgba)
    if "gray" in name:                                       # at most 256 colours: both files are coded, the smaller kept
        assert st["palette"] is not None and len(out) == min(st["sizes"])
    else:
        assert st["palette"] is None and out == OV.webp_lossless_encode(rgba)


def test_animation_frames_match_the_twin(pal, OP):
    from PIL import Image
    from oracle import webp_anim as OW
    rng = np.random.default_rng(2)
    cols = rng.integers(0, 256, (6, 3), dtype=np.uint8)
    frames = []
    for k in range(4):
        idx = np.zeros((48, 70), np.int64)
        idx[8 + 3 * k:30 + 3 * k, 10 + 5 * k:40 + 5 * k] = 1 + k
        idx[::9] = 5
        frames.append(Image.fromarray(cols[idx]))
    b = io.BytesIO()
    frames[0].save(b, "WEBP", save_all=True, append_images=frames[1:], lossless=True, duration=80, loop=0)
    data = b.getvalue()
    assert pal.set_webp_anim(1) == 0
    try:
        out = pal.compress_in_memory(data, _params(pal))
    finally:
        pal.set_webp_anim(0)
    canv, durs, _, _ = pal.webp_anim_decode(data)
    tf = OW.frames(canv, durs)
    top = wc._chunks(out)
    anmf = [p for t, p in top if t == b"ANMF"]
    assert len(anmf) == len(tf)
    for (k, (x, y, w, h), _), p in zip(tf, anmf):
        want = [t for t in wc._chunks(OP.webp_palette_encode(canv[k, y:y + h, x:x + w])) if t[0] == b"VP8L"]
        assert wc._chunks(p, 16) == want


def test_4k_flat_art_is_smaller(pal, OP, OV):
    img = synth(2160, 3840, 3, seed=7, kind="flat")
    src = _webp(img, lossless=True, method=0)
    px = _decoded_rgba(pal, src)
    on = pal.compress_in_memory(src, _params(pal))
    pal.set_webp_palette(0)
    off = pal.compress_in_memory(src, _params(pal))
    pal.set_webp_palette(1)
    assert off == OV.webp_lossless_encode(px)
    _check(on, OP, px)
    assert len(on) < len(off)


def test_photograph_keeps_todays_bytes(pal, OV):
    img = synth(720, 1280, 3, seed=3, kind="photo")
    src = _webp(img, lossless=True, method=0)
    on = pal.compress_in_memory(src, _params(pal))
    pal.set_webp_palette(0)
    off = pal.compress_in_memory(src, _params(pal))
    pal.set_webp_palette(1)
    assert on == off == OV.webp_lossless_encode(_decoded_rgba(pal, src))


def _mixed_sources():
    return [_webp(synth(h, w, 3, seed=h, kind=k), lossless=True)
            for h, w, k in ((400, 600, "flat"), (1, 1, "flat"), (33, 17, "photo"), (400, 600, "photo"), (5, 900, "flat"), (260, 3, "flat"))]


def test_repeated_calls_of_different_sizes(pal, OP):
    srcs = _mixed_sources()
    want = [OP.webp_palette_encode(_decoded_rgba(pal, s)) for s in srcs]
    for _ in range(2):
        assert [pal.compress_in_memory(s, _params(pal)) for s in srcs] == want


def test_threads_and_batch_give_the_twins_bytes(pal, OP):
    srcs = _mixed_sources() * 3
    want = [OP.webp_palette_encode(_decoded_rgba(pal, s)) for s in srcs]
    with ThreadPoolExecutor(6) as ex:
        assert list(ex.map(lambda s: pal.compress_in_memory(s, _params(pal)), srcs)) == want
    res = pal.compress_batch(srcs, _params(pal), n_threads=4)
    assert [r[1] for r in res] == [0] * len(srcs)
    assert [r[0] for r in res] == want


def test_switch_off_writes_todays_bytes(L, OV):
    assert L.lib().b200_init_device(0) == 0
    assert L.set_webp_palette(0) == 0
    for src in _mixed_sources():
        assert L.compress_in_memory(src, _params(L)) == OV.webp_lossless_encode(_decoded_rgba(L, src))
