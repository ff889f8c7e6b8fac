"""The lossless WebP (VP8L) palette kernels as the device runs them (csrc/vp8l_palette.cu, emulated serially by
tests/emul/vp8l_palette_emul.cpp through csrc/vp8l_palette_core.h: per-CTA colour sets with the overflow exit, the merge into one
global set, the bitonic sort, the bundling) equal a numpy restatement of the rule: the palette is np.unique of the ARGB words, an
image of more than 256 colours has none, and each packed pixel holds 1 << xbits indices by shifts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
CTA_PIXELS = 4096


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libvp8l_palette_emul.so")
    srcs = [os.path.join(EMUL_DIR, "vp8l_palette_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "vp8l_palette_core.h"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "vp8l_enc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, srcs[0]])
    return C.CDLL(so)


def run(emul, img):
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape[:2]
    info = np.zeros(258, np.uint32)
    packed = np.zeros(w * h, np.uint32)
    pw = C.c_int()
    stats = np.zeros(3, np.int32)
    emul.emul_vp8l_palette(img.ctypes.data_as(C.c_void_p), w, h, info.ctypes.data_as(C.c_void_p), packed.ctypes.data_as(C.c_void_p),
                           C.byref(pw), stats.ctypes.data_as(C.c_void_p))
    if info[1]:
        return None, None, stats
    k = int(info[0])
    return info[2:2 + k].copy(), packed[:pw.value * h].reshape(h, pw.value), stats


def numpy_palette(img):
    """(palette, packed image), or (None, None) over 256 colours"""
    img = img.astype(np.uint32)
    argb = (img[..., 3] << 24) | (img[..., 0] << 16) | (img[..., 1] << 8) | img[..., 2]
    pal = np.unique(argb)
    if len(pal) > 256:
        return None, None
    k = len(pal)
    xbits = 3 if k <= 2 else 2 if k <= 4 else 1 if k <= 16 else 0
    per = 1 << xbits
    h, w = argb.shape
    wp = (w + per - 1) >> xbits
    idx = np.zeros((h, wp * per), np.uint32)
    idx[:, :w] = np.searchsorted(pal, argb)
    bundle = np.zeros((h, wp), np.uint32)
    for j in range(per):
        bundle |= idx[:, j::per] << np.uint32(j * (8 >> xbits))
    return pal.astype(np.uint32), (np.uint32(0xFF000000) | (bundle << np.uint32(8))).astype(np.uint32)


def image(h, w, k, seed, last_only=False):
    """h x w RGBA holding exactly min(k, h * w) colours; last_only: the k-th colour only in the last pixel"""
    rng = np.random.default_rng(seed)
    cols = rng.integers(0, 256, (k, 4), dtype=np.uint8)
    while len(np.unique(cols.view(np.uint32))) < k:
        cols = rng.integers(0, 256, (k, 4), dtype=np.uint8)
    n = h * w
    m = k - 1 if last_only else k
    idx = rng.integers(0, m, n)
    if n >= m:
        idx[:m] = rng.permutation(m)
    if last_only:
        idx[-1] = k - 1
    return cols[idx].reshape(h, w, 4)


SHAPES = [(1, 1), (1, 37), (53, 1), (1, 16383), (16383, 1), (61, 83), (300, 200)]
COUNTS = [1, 2, 3, 4, 5, 16, 17, 255, 256, 257]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[1]}x{s[0]}")
@pytest.mark.parametrize("k", COUNTS)
def test_palette_and_packing_equal_numpy(emul, shape, k):
    h, w = shape
    img = image(h, w, k, seed=k * 7 + w)
    pal, packed, _ = run(emul, img)
    want_pal, want_packed = numpy_palette(img)
    if want_pal is None:
        assert pal is None
        return
    assert np.array_equal(pal, want_pal)
    assert np.array_equal(packed, want_packed)


@pytest.mark.parametrize("shape", [(1, 16383), (16383, 1), (300, 200)], ids=lambda s: f"{s[1]}x{s[0]}")
def test_257th_colour_only_in_the_last_pixel(emul, shape):
    h, w = shape
    img = image(h, w, 257, seed=3, last_only=True)
    assert run(emul, img)[0] is None
    img[-1, -1] = img[0, 0]                                   # 256 colours: the same image has a palette
    pal, packed, _ = run(emul, img)
    want_pal, want_packed = numpy_palette(img)
    assert len(want_pal) == 256 and np.array_equal(pal, want_pal) and np.array_equal(packed, want_packed)


def test_overflow_inside_one_cta_stops_the_rest(emul):
    # the first CTA's pixels alone hold more than 256 colours: it stops inside its steps, every later CTA at entry
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (40, 1000, 4), dtype=np.uint8)
    pal, _, stats = run(emul, img)
    nctas = -(-img.shape[0] * img.shape[1] // CTA_PIXELS)
    assert pal is None
    assert list(stats) == [0, 1, nctas - 1]


def test_overflow_across_ctas_is_found_by_the_merge(emul):
    # each CTA holds 200 colours of its own: no CTA overflows alone, the merge of the second pushes the global count past 256
    rng = np.random.default_rng(6)
    cols = np.unique(rng.integers(0, 1 << 32, 2000, dtype=np.uint64).astype(np.uint32))[:600]
    rgba = cols.view(np.uint8).reshape(-1, 4)
    idx = np.concatenate([rng.integers(0, 200, CTA_PIXELS) + 200 * c for c in range(3)])
    img = rgba[idx].reshape(3, CTA_PIXELS, 4)
    pal, _, stats = run(emul, img)
    assert pal is None
    assert list(stats) == [2, 0, 1]


def test_many_ctas_with_few_colours_merge_to_one_palette(emul):
    # 256 colours spread over 103 CTAs, half of them fully transparent with distinct RGB (colours in their own right)
    img = image(700, 600, 256, seed=9)
    cols = np.unique(img.reshape(-1, 4), axis=0)
    img[..., 3] = np.where(np.isin(img[..., 0], cols[::2, 0]), 0, img[..., 3])
    want_pal, want_packed = numpy_palette(img)
    assert want_pal is not None and (want_pal >> 24 == 0).sum() > 1
    pal, packed, stats = run(emul, img)
    assert np.array_equal(pal, want_pal) and np.array_equal(packed, want_packed)
    assert stats[0] == -(-700 * 600 // CTA_PIXELS) and stats[1] == stats[2] == 0
