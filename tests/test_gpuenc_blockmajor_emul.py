"""CPU checks of the device encoder's block-major passes (tests/emul/gpuenc_blockmajor_emul.cpp): each component's scan visits
reach every unit of every scan once, with ge::locate's block and DC predecessor, and symbols counted into / looked up in the
on-chip table slots give the scan-major histograms, bit lengths and bit buffer.  Golden files, every sampling geometry of
tests/jpeg_geometry.py, and coefficient patterns at the run-length and magnitude edges, sequential and progressive."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_geometry as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
INPUTS = ["in_420_base_355x237.jpg", "in_420_prog_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg",
          "in_gray_base_355x237.jpg", "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"]
CASES = [(name, w, h) for name, f in G.GEOMETRIES.items() for (w, h) in G.sizes_for(f)]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libgpuenc_blockmajor_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gpuenc_blockmajor_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_host.cpp"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_plan.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-o", so, srcs[0], srcs[1]])
    return C.CDLL(so)


def check(emul, data):
    for prog in (0, 1):
        assert emul.emul_blockmajor_check(data, C.c_size_t(len(data)), prog) == 0, prog


def _layout(L, w, h, ncomp, factors=None):
    lay = L.JpegLayout()
    lay.width, lay.height, lay.ncomp = w, h, ncomp
    off = 0
    for c in range(ncomp):
        lay.hs[c] = lay.vs[c] = 1
        lay.bw[c] = lay.rbw[c] = -(-w // 8)
        lay.bh[c] = lay.rbh[c] = -(-h // 8)
        lay.comp_offset[c] = off
        off += lay.bw[c] * lay.bh[c] * 64
        for k in range(64):
            lay.qt[c][k] = 1
    lay.total_coefs = off
    return lay


@pytest.mark.parametrize("name", INPUTS)
def test_golden(emul, golden, name):
    check(emul, golden(name))


@pytest.mark.parametrize("name,w,h", CASES)
def test_sampling_geometries(emul, name, w, h):
    check(emul, G.make_jpeg(w, h, G.GEOMETRIES[name], False))


def test_edge_blocks(L, emul):
    """Empty and all-non-zero blocks, extreme coefficients (a DC of -32768; AC symbols carry at most 15 magnitude bits, so AC
    values stop at +-32767), zero runs of 15, 16, 31, 32, 47 and 48 ahead of a non-zero coefficient (the ZRL edges), refinement
    blocks whose last newly non-zero coefficient is at 63, and a component of 9 x 7 = 63 blocks (not a multiple of a warp or a
    CTA)."""
    lay = _layout(L, 72, 56, 3)
    co = np.zeros(lay.total_coefs, dtype=np.int16)
    blocks = co.reshape(-1, 64)
    rng = np.random.default_rng(7)
    blocks[:, 0] = rng.integers(-2000, 2000, size=len(blocks))
    n = 0
    for run in (15, 16, 31, 32, 47, 48):
        for v in (1, 2, 3, -5):
            blocks[n, 1 + run] = v
            blocks[n + 1, 1] = v
            blocks[n + 1, 2 + run] = -v
            n += 2
    blocks[n] = rng.choice([-3, -2, -1, 1, 2, 3, 700, -32767, 32767], size=64); blocks[n, 0] = -32768; n += 1
    blocks[n, 0] = -32768; blocks[n + 1, 0] = 32767; n += 2                  # the largest DC difference
    blocks[n, 63] = 1; blocks[n, 5] = 3; n += 1                                # refinement: new coefficient at Se
    blocks[n, 63] = -1; blocks[n, 1:63] = 2; n += 1
    blocks[n, 1:] = -32767; n += 1
    blocks[n, 1:] = 1; n += 1
    mix = rng.random((len(blocks) - n, 64))
    blocks[n:, 1:] = np.where(mix[:, 1:] < 0.2, rng.integers(-9, 10, size=mix[:, 1:].shape), 0)
    check(emul, L.jpeg_encode_coefficients(lay, co, 1))
    check(emul, L.jpeg_encode_coefficients(lay, co, 0))
