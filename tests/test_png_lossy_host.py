"""Lossy PNG quantiser, CPU side: invariants of the scalar twin (oracle/png_quant_oracle.c over csrc/png_quant_core.h), its quality
against Pillow's median cut with Floyd-Steinberg dithering, and the C declarations of the opt-in header."""
import os
import subprocess

import numpy as np
import pytest

from oracle.png_quant import png_quantize
from pngutil import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rgba_of(img):
    if img.shape[2] == 4:
        return img
    return np.concatenate([img, np.full(img.shape[:2] + (1,), 255, np.uint8)], axis=2)


def photos():
    return [rgba_of(synth(96, 128, 3, seed=s)) for s in range(3)]


def soft_alpha(h=48, w=64, seed=3):
    img = synth(h, w, 4, seed=seed)
    img[:, : w // 4, 3] = 0                                  # a fully transparent band with varied RGB underneath
    return img


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 10 * np.log10(255.0 ** 2 / mse) if mse else float("inf")


@pytest.mark.parametrize("q", [1, 40, 80, 100])
@pytest.mark.parametrize("kind", ["photo", "alpha"])
def test_palette_and_indices_are_in_range(kind, q):
    img = photos()[0] if kind == "photo" else soft_alpha()
    pal, idx = png_quantize(img, q)
    assert 1 <= len(pal) <= 256
    assert idx.shape == img.shape[:2] and int(idx.max()) < len(pal)
    opaque = pal[:, 3] == 255
    assert not np.any(opaque[:-1] & ~opaque[1:]), "entries that are not opaque come first"


def test_few_colours_come_back_exactly():
    img = rgba_of(synth(40, 56, 3, seed=1, kind="flat"))
    img[0, 0] = (1, 2, 3, 0); img[1, 1] = (9, 9, 9, 0)     # two transparent values stay distinct on the exact path
    assert len(np.unique(img.reshape(-1, 4), axis=0)) <= 256
    for q in (1, 80):
        pal, idx = png_quantize(img, q)
        assert np.array_equal(pal[idx], img)


def photo_with_hole():
    img = photos()[0].copy()
    img[40:44, 60:64] = (200, 30, 90, 0)                      # a small fully transparent hole in an opaque photograph
    return img


def test_transparent_pixels_share_one_transparent_entry():
    for img in (soft_alpha(), photo_with_hole()):
        for q in (1, 40, 80, 100):
            pal, idx = png_quantize(img, q)
            assert set(np.unique(idx[img[:, :, 3] == 0])) == {0}
            assert tuple(pal[0]) == (0, 0, 0, 0) and not (pal[1:, 3] == 0).any()


@pytest.mark.parametrize("q", [1, 10, 20, 30, 80])
def test_a_transparent_hole_stays_transparent_and_the_rest_opaque(q):
    img = photo_with_hole()
    pal, idx = png_quantize(img, q)
    out = pal[idx]
    hole = img[:, :, 3] == 0
    assert (out[hole, 3] == 0).all()
    assert (out[~hole, 3] == 255).all()


def test_lower_quality_never_gives_more_colours():
    for img in photos()[:2] + [soft_alpha()]:
        counts = [len(png_quantize(img, q)[0]) for q in (1, 10, 25, 40, 55, 70, 80, 90, 100)]
        assert counts == sorted(counts), counts


def test_photo_at_q100_uses_256_colours():
    for img in photos():
        assert len(png_quantize(img, 100)[0]) == 256


def test_quality_at_q80_is_not_below_pillow_median_cut():
    # Pillow here is built without libimagequant, so imagequant itself cannot be the yardstick; its median cut with Floyd-Steinberg
    # dithering is.  Image.quantize(256, method=MEDIANCUT, dither=FLOYDSTEINBERG) does not dither (Pillow applies `dither` only
    # when a palette is given), so the median-cut palette is applied again with the dithering switched on: dithered against dithered.
    from PIL import Image
    for img in photos():
        pal, idx = png_quantize(img, 80)
        ours = psnr(pal[idx], img)
        rgb = Image.fromarray(img[:, :, :3])
        mc = rgb.quantize(256, method=Image.Quantize.MEDIANCUT, dither=Image.Dither.FLOYDSTEINBERG)
        theirs = psnr(rgba_of(np.asarray(rgb.quantize(palette=mc, dither=Image.Dither.FLOYDSTEINBERG).convert("RGB"))), img)
        assert ours >= theirs, (ours, theirs)


def blurred_error(a, b, r=2):
    """mean absolute error after a (2r+1)^2 box blur of both: the low-frequency error dithering exists to remove (banding)"""
    d = a.astype(np.float64) - b.astype(np.float64)
    k = 2 * r + 1
    c = np.cumsum(np.cumsum(np.pad(d, ((1, 0), (1, 0), (0, 0))), 0), 1)
    box = (c[k:, k:] - c[:-k, k:] - c[k:, :-k] + c[:-k, :-k]) / (k * k)
    return np.abs(box).mean()


def test_dithering_removes_banding_on_a_gradient():
    h, w = 64, 256
    yy, xx = np.mgrid[:h, :w]
    img = rgba_of(np.stack([xx * 255 // (w - 1), 64 + yy, 200 - xx // 4], -1).astype(np.uint8))
    pal, idx = png_quantize(img, 40)
    d = ((img[:, :, None, :].astype(np.int64) - pal[None, None].astype(np.int64)) ** 2).sum(-1)
    nearest = pal[d.argmin(-1)]                               # the same palette without dithering
    assert blurred_error(pal[idx], img) < 0.75 * blurred_error(nearest, img)


def test_opt_in_header_is_c99(tmp_path):
    src = tmp_path / "png_lossy_abi.c"
    src.write_text('#include "b200_caesium_png_lossy.h"\n'
                   "typedef void (*fn)(void);\n"
                   "int main(void) { fn f[2] = {(fn)b200_set_png_lossy, (fn)b200_png_quantize}; return f[0] == 0 || f[1] == 0; }\n")
    pkg = os.path.join(ROOT, "caesium-clt_b200")
    exe = str(tmp_path / "png_lossy_abi")
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe,
                        "-L", pkg, "-lb200caesium", "-Wl,-rpath," + pkg], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([exe]).returncode == 0
