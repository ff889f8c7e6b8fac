"""CPU checks of the device encoder's statistics and bit-writer shortcuts (tests/emul/gpuenc_stats_emul.cpp): inline symbols
counted in the classify pass plus EOBn symbols counted where the EOB groups are recorded equal the histogram of every symbol,
including runs that overflow the EOBRUN counter or the correction-bit buffer; and interior words written with plain stores
equal the words written with OR only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
INPUTS = ["in_420_base_355x237.jpg", "in_420_prog_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg",
          "in_gray_base_355x237.jpg", "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libgpuenc_stats_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gpuenc_stats_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_host.cpp"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_plan.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-o", so, srcs[0], srcs[1]])
    return C.CDLL(so)


def check(emul, data):
    for prog in (0, 1):
        assert emul.emul_stats_check(data, C.c_size_t(len(data)), prog) == 0, prog


def _layout(L, w, h, ncomp):
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
def test_split_statistics_and_plain_stores(emul, golden, name):
    check(emul, golden(name))


def test_eobrun_counter_overflow(L, emul):
    """> 0x7FFF consecutive blocks with empty AC bands: the groups come from the overflow replay."""
    lay = _layout(L, 2048, 2048, 1)
    co = np.zeros(lay.total_coefs, dtype=np.int16)
    co[::64] = 5
    co[64 * 50000 + 9] = 3
    check(emul, L.jpeg_encode_coefficients(lay, co, 1))


def test_correction_bit_buffer_overflow(L, emul):
    """Long runs of correction-only blocks in the refinement scans force mid-run flushes (> 937 pending bits)."""
    rng = np.random.default_rng(29)
    lay = _layout(L, 512, 384, 3)
    co = np.zeros(lay.total_coefs, dtype=np.int16)
    blocks = co.reshape(-1, 64)
    blocks[:, 0] = rng.integers(-60, 60, size=len(blocks))
    for b in range(len(blocks)):
        kind = rng.random()
        if kind < 0.85:
            idx = rng.choice(np.arange(1, 64), size=int(rng.integers(12, 45)), replace=False)
            blocks[b, idx] = rng.choice([-7, -4, -3, -2, 2, 3, 5, 6], size=len(idx))
        elif kind < 0.9:
            idx = rng.choice(np.arange(1, 64), size=10, replace=False)
            blocks[b, idx] = rng.choice([-1, 1, -3, 2, 9], size=10)
    check(emul, L.jpeg_encode_coefficients(lay, co, 1))


def test_dense_blocks(L, emul):
    """Dense blocks: long bit ranges, so most words of a block are interior ones."""
    rng = np.random.default_rng(31)
    lay = _layout(L, 256, 128, 3)
    co = rng.integers(-300, 301, size=lay.total_coefs).astype(np.int16)
    check(emul, L.jpeg_encode_coefficients(lay, co, 0))
