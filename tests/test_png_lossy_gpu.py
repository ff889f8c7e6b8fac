"""Lossy PNG on the device (b200_set_png_lossy): the quantiser against its scalar twin bit for bit, and every call that reaches it --
compress, JPEG / WebP -> PNG conversion, compress_to_size, batch -- decoding to the twin's palette applied to the twin's indices."""
import io
import struct
import zlib

import numpy as np
import pytest

from oracle.png_quant import png_quantize as oracle_quantize
from pngutil import chunk, frame_png, pil_pixels, pil_png, synth

pytestmark = pytest.mark.gpu

FMT_JPEG, FMT_PNG, FMT_WEBP = 0, 1, 3


@pytest.fixture
def lossy(L):
    assert L.set_png_lossy(True) == 0
    yield L
    L.set_png_lossy(False)


def rgba_of(img):
    img = np.asarray(img, np.uint8)
    if img.ndim == 2:
        img = img[:, :, None]
    if img.shape[2] == 1:
        return np.concatenate([np.repeat(img, 3, 2), np.full(img.shape[:2] + (1,), 255, np.uint8)], 2)
    if img.shape[2] == 2:
        return np.concatenate([np.repeat(img[:, :, :1], 3, 2), img[:, :, 1:]], 2)
    if img.shape[2] == 3:
        return np.concatenate([img, np.full(img.shape[:2] + (1,), 255, np.uint8)], 2)
    return img


def soft_alpha(h=48, w=64, seed=3):
    img = synth(h, w, 4, seed=seed)
    img[:, : w // 4, 3] = 0
    return img


def photo_with_hole():
    img = rgba_of(synth(96, 128, 3, seed=0))
    img[40:44, 60:64] = (200, 30, 90, 0)
    return img


def decoded_rgba(data):
    return np.asarray(pil_pixels(data).convert("RGBA"))


def lossy_params(L, q=80, level=3):
    p = L.default_params()
    p.png_optimize, p.png_quality, p.png_optimization_level = 0, q, level
    return p


def expect(rgba, q):
    pal, idx = oracle_quantize(rgba, q)
    return pal[idx]


CASES = {
    "photo": lambda: rgba_of(synth(96, 128, 3, seed=0)),
    "flat": lambda: rgba_of(synth(40, 56, 3, seed=1, kind="flat")),
    "soft_alpha": soft_alpha,
    "grey": lambda: rgba_of(synth(33, 45, 1, seed=2)),
    "noise_1x1": lambda: rgba_of(synth(1, 1, 3, seed=4, kind="noise")),
    "noise_3x3": lambda: rgba_of(synth(3, 3, 4, seed=5, kind="noise")),
    "odd_37x29": lambda: rgba_of(synth(29, 37, 3, seed=6, kind="noise")),
    "tall_200x33": lambda: rgba_of(synth(200, 33, 3, seed=7)),
    "photo_with_hole": photo_with_hole,
    "all_transparent": lambda: np.concatenate([synth(20, 30, 3, seed=12, kind="noise"), np.zeros((20, 30, 1), np.uint8)], 2),
}


@pytest.mark.parametrize("q", [1, 40, 80, 100])
@pytest.mark.parametrize("case", sorted(CASES))
def test_quantize_equals_the_oracle(L, case, q):
    img = CASES[case]()
    pal, idx = L.png_quantize(img, q)
    opal, oidx = oracle_quantize(img, q)
    assert np.array_equal(pal, opal)
    assert np.array_equal(idx, oidx)


@pytest.mark.parametrize("level", [0, 3, 6])
def test_compress_decodes_to_the_oracle(lossy, level):
    L = lossy
    for img in (synth(96, 128, 3, seed=0), soft_alpha(), synth(40, 56, 3, seed=1, kind="flat")):
        src = pil_png(img)
        out = L.compress_in_memory(src, lossy_params(L, 80, level))
        assert np.array_equal(decoded_rgba(out), expect(rgba_of(img), 80))


@pytest.mark.parametrize("q", [1, 10, 30])
def test_low_quality_keeps_a_hole_transparent_and_the_rest_opaque(lossy, q):
    img = photo_with_hole()
    a = decoded_rgba(lossy.compress_in_memory(pil_png(img), lossy_params(lossy, q)))[:, :, 3]
    hole = img[:, :, 3] == 0
    assert (a[hole] == 0).all() and (a[~hole] == 255).all()


def test_lossy_is_smaller_than_lossless_on_photos(lossy):
    L = lossy
    for seed in range(3):
        src = pil_png(synth(128, 160, 3, seed=seed))
        lossless = L.default_params(); lossless.png_optimize = 1
        assert len(L.compress_in_memory(src, lossy_params(L))) < len(L.compress_in_memory(src, lossless))


def test_two_calls_give_identical_bytes(lossy):
    src = pil_png(soft_alpha(64, 96))
    p = lossy_params(lossy, 60)
    assert lossy.compress_in_memory(src, p) == lossy.compress_in_memory(src, p)


def _sources():
    """(name, PNG bytes, the RGBA the quantiser sees)"""
    out = []
    g = synth(33, 45, 1, seed=2)
    out.append(("grey", pil_png(g), rgba_of(g)))
    la = synth(30, 41, 2, seed=8)
    out.append(("grey_alpha", pil_png(la), rgba_of(la)))
    rgb = synth(31, 47, 3, seed=9)
    # 16 bits per sample: the high byte counts
    s16 = rgb.astype(np.uint16) * 256 + (np.arange(rgb.size).reshape(rgb.shape) % 251).astype(np.uint16)
    rows = b"".join(b"\x00" + s16[y].astype(">u2").tobytes() for y in range(s16.shape[0]))
    out.append(("rgb16", frame_png(47, 31, 16, 2, zlib.compress(rows)), rgba_of(rgb)))
    # colour key: tRNS on an 8-bit RGB image
    key = rgb.copy(); key[5:9, 3:20] = (10, 20, 30)
    rows = b"".join(b"\x00" + key[y].tobytes() for y in range(key.shape[0]))
    keyed = rgba_of(key); keyed[5:9, 3:20, 3] = 0
    out.append(("rgb_key", frame_png(47, 31, 8, 2, zlib.compress(rows), chunk(b"tRNS", struct.pack(">HHH", 10, 20, 30))), keyed))
    # sub-byte and 16-bit grey, with and without a colour key (the key compares the full sample)
    for bd in (1, 2, 4, 16):
        top = (1 << bd) - 1
        v = (np.add.outer(np.arange(23), np.arange(37)) * 7 + 3 * np.arange(37)) % (top + 1)
        if bd == 16:
            rows = b"".join(b"\x00" + v[y].astype(">u2").tobytes() for y in range(v.shape[0]))
            g8 = (v >> 8).astype(np.uint8)
        else:
            per = 8 // bd
            packed = []
            for y in range(v.shape[0]):
                row = bytearray((v.shape[1] * bd + 7) // 8)
                for x in range(v.shape[1]):
                    row[x // per] |= int(v[y, x]) << (8 - bd - (x % per) * bd)
                packed.append(b"\x00" + bytes(row))
            rows = b"".join(packed)
            g8 = (v * 255 // top).astype(np.uint8)
        key = int(v[3, 5])
        for keyed in (False, True):
            extra = chunk(b"tRNS", struct.pack(">H", key)) if keyed else b""
            rgba = rgba_of(g8)
            if keyed:
                rgba = rgba.copy(); rgba[v == key, 3] = 0
            out.append((f"grey{bd}{'_key' if keyed else ''}", frame_png(37, 23, bd, 0, zlib.compress(rows), extra), rgba))
    # palette source with tRNS (a palette has at most 256 entries, so it takes the exact path after expansion)
    from PIL import Image
    pim = Image.fromarray(synth(29, 35, 3, seed=10)).quantize(200)
    b = io.BytesIO(); pim.save(b, format="PNG", transparency=bytes(range(0, 200)))
    out.append(("palette_trns", b.getvalue(), np.asarray(Image.open(io.BytesIO(b.getvalue())).convert("RGBA"))))
    # palette source
    pim = Image.fromarray(synth(29, 35, 3, seed=10)).quantize(64)
    b = io.BytesIO(); pim.save(b, format="PNG")
    out.append(("palette", b.getvalue(), np.asarray(pim.convert("RGBA"))))
    return out


def test_every_source_colour_type(lossy):
    for name, src, rgba in _sources():
        out = lossy.compress_in_memory(src, lossy_params(lossy, 40))
        assert np.array_equal(decoded_rgba(out), expect(rgba, 40)), name


def test_jpeg_to_png_with_resize(lossy, golden):
    L = lossy
    data = golden("in_420_base_355x237.jpg")
    ref = L.default_params(); ref.png_optimize = 1; ref.width = 200
    rgba = decoded_rgba(L.convert_in_memory(data, ref, FMT_PNG))
    p = lossy_params(L, 70); p.width = 200
    assert np.array_equal(decoded_rgba(L.convert_in_memory(data, p, FMT_PNG)), expect(rgba, 70))


def test_webp_to_png_keeps_alpha(lossy):
    L = lossy
    webp = L.convert_in_memory(pil_png(soft_alpha(40, 52)), L.default_params(), FMT_WEBP)
    ref = L.default_params(); ref.png_optimize = 1
    rgba = decoded_rgba(L.convert_in_memory(webp, ref, FMT_PNG))
    assert (rgba[:, :, 3] < 255).any()
    assert np.array_equal(decoded_rgba(L.convert_in_memory(webp, lossy_params(L, 80), FMT_PNG)), expect(rgba, 80))


def test_compress_to_size_follows_the_bisection(lossy):
    L = lossy
    src = pil_png(synth(96, 128, 3, seed=11))
    sizes = {}

    def size_of(q):
        if q not in sizes:
            sizes[q] = len(L.compress_in_memory(src, lossy_params(L, q)))
        return sizes[q]

    limit = (size_of(1) + size_of(100)) // 2
    lo, hi, q, best, best_q = 1, 100, 80, 0, None
    for _ in range(10):
        if lo > hi:
            break
        sz = size_of(q)
        if sz <= limit:
            if sz > best:
                best, best_q = sz, q
            if limit - sz <= limit // 50:
                break
            lo = q + 1
        else:
            hi = q - 1
        q = (lo + hi) // 2
    p = lossy_params(L, 80)
    out = L.compress_to_size_in_memory(src, p, limit)
    assert p.png_quality == best_q
    assert out == L.compress_in_memory(src, lossy_params(L, p.png_quality))


def test_batch_equals_single_calls(lossy):
    L = lossy
    srcs = [pil_png(synth(50 + 7 * i, 60, 3, seed=i)) for i in range(4)] + [pil_png(soft_alpha())]
    p = lossy_params(L, 70)
    res = L.compress_batch(srcs, p, n_threads=3)
    for s, (data, code, msg) in zip(srcs, res):
        assert code == 0, msg
        assert data == L.compress_in_memory(s, p)


def test_switch_off_still_refuses(L, golden):
    src = pil_png(synth(16, 16, 3))
    p = lossy_params(L)
    for call in (lambda: L.compress_in_memory(src, p), lambda: L.compress_to_size_in_memory(src, p, 10),
                 lambda: L.convert_in_memory(golden("in_420_base_355x237.jpg"), p, FMT_PNG)):
        with pytest.raises(L.B200Error) as e:
            call()
        assert e.value.code == 3
    assert L.lib().b200_set_png_lossy(2) != 0
