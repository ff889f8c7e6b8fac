"""The lossless WebP (VP8L) palette variant's oracle twin (oracle/vp8l_palette_oracle.c) on the CPU: every palette file it writes
decodes through libwebp (Pillow) and through the project's own VP8L decoder to exactly the source pixels, the file it keeps is never
larger than the encoder's file without the palette and is that very file over 256 colours, and it is strictly smaller on flat
images.  Also the switch's C header and its refusals."""
import io
import os
import re
import subprocess

import numpy as np
import pytest

from pngutil import synth
from webp_palette_cases import coloured, sprite_sheet, two_colour_bitmap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caesium-clt_b200")


@pytest.fixture(scope="module")
def OV(O):
    from oracle import vp8l
    return vp8l


@pytest.fixture(scope="module")
def OP(O):
    """the palette variant's twin (oracle/vp8l_palette.py over oracle/vp8l_palette_oracle.c)"""
    from oracle import vp8l_palette
    return vp8l_palette


def _pil_rgba(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    assert im.format == "WEBP"
    return np.asarray(im.convert("RGBA"))


def _own_rgba(L, data):
    rgb, a = L.webp_decode_rgba(data)
    if a is None:
        a = np.full(rgb.shape[:2], 255, np.uint8)
    return np.concatenate([rgb, a[:, :, None]], axis=2)


COUNTS = [1, 2, 3, 4, 5, 16, 17, 255, 256, 257]
# widths around every bundle size (8, 4, 2 indices per pixel): multiples and not
SHAPES = [(1, 1), (1, 37), (29, 1), (23, 45), (17, 64), (9, 257)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[1]}x{s[0]}")
@pytest.mark.parametrize("k", COUNTS)
@pytest.mark.parametrize("alpha", ["opaque", "translucent", "hidden"])
def test_palette_files_decode_exactly_and_the_kept_file_is_never_larger(L, OV, OP, shape, k, alpha):
    h, w = shape
    img = coloured(h, w, k, seed=1000 * k + 10 * w + h, alpha=alpha)
    st = OP.webp_palette_stages(img)
    plain = OV.webp_lossless_encode(img)
    assert st["sizes"][0] == len(plain)
    ncol = len(np.unique(img.reshape(-1, 4).view(np.uint32)))
    if ncol > 256:
        assert st["palette"] is None and st["sizes"][1] == 0
        assert st["file"] == plain                           # over 256 colours: the encoder's file, byte for byte
        return
    assert len(st["palette"]) == ncol and np.all(np.diff(st["palette"].astype(np.int64)) > 0)
    pf = st["palette_file"]
    assert len(pf) == st["sizes"][1]
    assert np.array_equal(_pil_rgba(pf), img), "libwebp decode of the palette file"
    assert np.array_equal(_own_rgba(L, pf), img), "own decode of the palette file"
    assert len(st["file"]) <= len(plain)
    assert st["file"] == (pf if len(pf) < len(plain) else plain)   # ties keep the file without the palette
    assert np.array_equal(_pil_rgba(st["file"]), img)


@pytest.mark.parametrize("case", ["flat", "bitmap", "sprite"])
def test_flat_images_are_strictly_smaller(OV, OP, case):
    img = {"flat": lambda: synth(300, 400, 3, seed=7, kind="flat"), "bitmap": lambda: two_colour_bitmap(250, 333),
           "sprite": lambda: sprite_sheet(256, 384)}[case]()
    st = OP.webp_palette_stages(img)
    plain = OV.webp_lossless_encode(img)
    assert st["palette"] is not None and len(st["file"]) < len(plain)
    assert st["file"] == st["palette_file"]
    assert np.array_equal(_pil_rgba(st["file"])[..., :img.shape[2]], img)


def test_photographs_keep_the_encoders_file(OV, OP):
    img = synth(120, 170, 3, seed=2, kind="photo")
    st = OP.webp_palette_stages(img)
    assert st["palette"] is None and st["file"] == OV.webp_lossless_encode(img)


def test_4k_flat_art_against_libwebp(OP):
    # 3840 x 2160 flat art (synth(..., kind="flat"), seed 7, 13 colours): the encoder's file without the palette is 15,366 B, with the
    # palette 7,594 B; libwebp (Pillow, lossless=True, method=4) writes 2,416 B -- it also predicts the index image and has a
    # stronger LZ77 search (DESIGN.md §4.7).
    from PIL import Image
    img = synth(2160, 3840, 3, seed=7, kind="flat")
    st = OP.webp_palette_stages(img)
    assert st["sizes"] == (15366, 7594) and len(st["file"]) == 7594
    b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", lossless=True, method=4)
    assert len(b.getvalue()) < len(st["file"])


def test_switch_refuses_other_values(L):
    assert L.set_webp_palette(2) != 0 and L.set_webp_palette(-1) != 0
    assert L.set_webp_palette(0) == 0


def test_header_is_c99_and_links(tmp_path):
    exe = str(tmp_path / "c_abi_webp_palette_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_webp_palette_check.c"), "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "webp palette c-abi ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_webp_palette.h")).read()
    declared = set(re.findall(r"^[a-z_0-9 ]+\b(b200_[a-z0-9_]+)\(", hdr, re.M))
    src = open(os.path.join(ROOT, "tests", "c_abi_webp_palette_check.c")).read()
    assert declared == {"b200_set_webp_palette"} and all("(fn)" + f in src for f in declared)
