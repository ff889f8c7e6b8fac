"""The lossless WebP (VP8L) analysis kernels as the device runs them (csrc/vp8l_kernels.cu, emulated serially by tests/emul/vp8l_emul.cpp
through csrc/vp8l_enc_core.h: tile scoring with the n log2 n table, the colour cache by per-chunk tables + carry + 32-pixel steps, the
copy search on bit arrays, the parse by pointer doubling) equal the oracle's plain loops: tile modes, cache hits and tokens."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")


@pytest.fixture(scope="module")
def OV(O):
    """the lossless WebP encoder twin (oracle/vp8l.py over oracle/vp8l_oracle.c)"""
    from oracle import vp8l
    return vp8l


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libvp8l_emul.so")
    srcs = [os.path.join(EMUL_DIR, "vp8l_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "vp8l_enc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emul_vp8l_stages.restype = C.c_size_t
    return lib


def _images():
    rng = np.random.default_rng(11)
    yy, xx = np.mgrid[0:120, 0:150]
    grad = np.stack([xx * 255 // 149, yy * 2, (xx + yy) % 256, np.full_like(xx, 255)], -1).astype(np.uint8)
    yield "gradient", grad, True
    yield "noise_alpha", rng.integers(0, 256, (40, 70, 4), dtype=np.uint8), True
    two = rng.integers(0, 2, (90, 77, 1), dtype=np.uint8) * np.array([[[200, 10, 30, 255]]], np.uint8) + 20
    yield "two_colours", two.astype(np.uint8), True
    tile = np.tile(rng.integers(0, 256, (6, 9, 4), dtype=np.uint8), (30, 25, 1)); tile[..., 3] = 255
    yield "tiled", tile, True
    flat = np.zeros((70, 300, 4), np.uint8); flat[..., 3] = 255; flat[20:40, 50:200] = (10, 200, 30, 255)
    yield "flat_long_runs", flat, False                   # copies of 4096 pixels, chunk ends inside runs
    yield "width1", rng.integers(0, 3, (300, 1, 4), dtype=np.uint8) * 60, True
    yield "width2", rng.integers(0, 3, (200, 2, 4), dtype=np.uint8) * 60, True
    yield "one_row", rng.integers(0, 3, (1, 300, 4), dtype=np.uint8) * 60, True
    yield "one_pixel", np.array([[[1, 2, 3, 4]]], np.uint8), True
    soft = np.zeros((64, 96, 4), np.uint8); soft[..., :3] = rng.integers(0, 256, (64, 96, 3)); soft[..., 3] = np.where(rng.random((64, 96)) < 0.5, 0, 255)
    yield "transparent_colours", soft, True


@pytest.mark.parametrize("case", list(_images()), ids=lambda c: c[0])
def test_device_shaped_stages_equal_the_oracle(emul, OV, case):
    _, img, check_def = case
    img = np.ascontiguousarray(img)
    h, w = img.shape[:2]
    n = w * h
    modes = np.zeros(((h + 15) // 16) * ((w + 15) // 16), np.uint8)
    hits = np.zeros((3, n), np.uint8)
    tok = np.zeros((n, 2), np.uint32)
    nt = emul.emul_vp8l_stages(img.ctypes.data_as(C.c_void_p), w, h, int(check_def), modes.ctypes.data_as(C.c_void_p),
                               hits.ctypes.data_as(C.c_void_p), tok.ctypes.data_as(C.c_void_p))
    assert nt != C.c_size_t(-1).value, "bit-array copy search differs from vp8l_best_copy"
    st = OV.webp_lossless_stages(img)
    assert np.array_equal(modes, st["modes"].reshape(-1)), "tile modes"
    assert np.array_equal(hits, st["hits"]), "colour-cache hits"
    assert np.array_equal(tok[:nt], st["tokens"]), "tokens"
