"""The lossless WebP (VP8L) bitstream as the encoder writes it (the oracle twin of the device encoder, oracle/vp8l_oracle.c, on the
rules of csrc/vp8l_enc_core.h): every file decodes to exactly its RGBA input through libwebp (Pillow) and through the project's own
decoder (b200_webp_decode_rgba) -- over content, sizes, alpha (colour under alpha 0 kept), every predictor mode, every cache size,
copies longer than one chunk, and widths whose distance codes clamp to 1."""
import io

import numpy as np
import pytest

from pngutil import synth


@pytest.fixture(scope="module")
def OV(O):
    """the lossless WebP encoder twin (oracle/vp8l.py over oracle/vp8l_oracle.c)"""
    from oracle import vp8l
    return vp8l


def _rgba(img):
    img = np.asarray(img, np.uint8)
    if img.shape[2] == 3:
        img = np.concatenate([img, np.full(img.shape[:2] + (1,), 255, np.uint8)], axis=2)
    return np.ascontiguousarray(img)


def _check(L, OV, img, **kw):
    from PIL import Image
    want = _rgba(img)
    st = OV.webp_lossless_stages(want, **kw)
    f = st["file"]
    assert f[:4] == b"RIFF" and f[8:16] == b"WEBPVP8L" and int.from_bytes(f[4:8], "little") == len(f) - 8
    translucent = bool((want[:, :, 3] != 255).any())
    assert bool(f[24] & 0x10) == translucent, "alpha_is_used"
    im = Image.open(io.BytesIO(f)); im.load()
    assert np.array_equal(np.asarray(im.convert("RGBA")), want), "libwebp decode"
    rgb, a = L.webp_decode_rgba(f)
    assert np.array_equal(rgb, want[:, :, :3]), "project decoder: colour"
    if translucent:
        assert np.array_equal(a, want[:, :, 3]), "project decoder: alpha"
    return st


def _content(kind, h, w, seed=0):
    rng = np.random.default_rng(seed)
    if kind in ("photo", "flat"):
        return synth(h, w, 3, seed=seed, kind=kind)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "gradient":
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + 2 * yy) % 256], -1).astype(np.uint8)
    if kind == "tiled":
        return np.tile(rng.integers(0, 256, (7, 5, 3), dtype=np.uint8), (h // 7 + 1, w // 5 + 1, 1))[:h, :w].copy()
    if kind == "two":
        return np.where(rng.random((h, w, 1)) < 0.3, np.array([250, 20, 40], np.uint8), np.array([5, 5, 90], np.uint8)).astype(np.uint8)
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["photo", "flat", "noise", "gradient", "tiled", "two"])
@pytest.mark.parametrize("h,w", [(1, 1), (300, 1), (1, 300), (9, 17), (37, 53), (65, 129)])
def test_round_trip_opaque(L, OV, kind, h, w):
    _check(L, OV, _content(kind, h, w, seed=h + w))


@pytest.mark.parametrize("kind", ["photo", "flat", "noise"])
def test_round_trip_with_alpha_keeps_colour_under_transparency(L, OV, kind):
    h, w = 61, 83
    rng = np.random.default_rng(5)
    rgb = _content(kind, h, w, seed=3)
    a = rng.integers(0, 256, (h, w), dtype=np.uint8)
    a[: h // 3] = 0                                         # alpha 0 over non-zero colour: exact mode keeps the colour
    a[h // 3: h // 2] = 255
    _check(L, OV, np.concatenate([rgb, a[:, :, None]], axis=2))


def test_round_trip_16383_wide(L, OV):
    img = _content("gradient", 2, 16383)
    _check(L, OV, img)


@pytest.mark.parametrize("mode", range(14))
def test_every_predictor_mode(L, OV, mode):
    rng = np.random.default_rng(mode)
    img = np.concatenate([_content("photo", 33, 47, seed=mode), rng.integers(0, 256, (33, 47, 1), dtype=np.uint8)], axis=2)
    st = _check(L, OV, img, force_mode=mode)
    assert (st["modes"] == mode).all()


@pytest.mark.parametrize("cand,bits", [(0, 0), (1, 6), (2, 8), (3, 10)])
def test_every_cache_size(L, OV, cand, bits):
    rng = np.random.default_rng(cand)
    img = _content("tiled", 120, 140, seed=1) ^ rng.integers(0, 2, (120, 140, 3), dtype=np.uint8)
    st = _check(L, OV, img, force_cache=cand)
    assert st["cache_bits"] == bits


def test_cache_chosen_when_it_pays(L, OV):
    # few colours in noisy order: a colour cache wins over plain literals, so the estimate must pick one
    rng = np.random.default_rng(2)
    pal = rng.integers(0, 256, (40, 3), dtype=np.uint8)
    st = _check(L, OV, pal[rng.integers(0, 40, (150, 160))])
    assert st["cache_bits"] > 0


def test_copies_longer_than_a_chunk(L, OV):
    img = np.zeros((40, 1000, 3), np.uint8); img[10:12, 100:900] = (1, 2, 3)
    st = _check(L, OV, img)
    lens = st["tokens"][:, 1] >> 8
    assert lens.max() == 4096                               # a whole chunk in one copy
    assert len(st["tokens"]) < 100


@pytest.mark.parametrize("w", [1, 2])
def test_narrow_images_with_clamped_distance_codes(L, OV, w):
    rng = np.random.default_rng(w)
    img = np.repeat(rng.integers(0, 3, (200, 1, 3), dtype=np.uint8) * 70, w, axis=1)
    img[50:120] = 9
    st = _check(L, OV, img)
    assert (st["tokens"][:, 1] != 0).any()

