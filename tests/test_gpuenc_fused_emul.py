"""CPU checks of the device encoder's scan sizes and single-pass emission (tests/emul/gpuenc_fused_emul.cpp): scan sizes from the
histograms (count x (code length + extra bits)) plus the refinement scans' correction bits equal the sum of the per-unit bit
lengths, and the bit buffer built from per-thread slots, CTA runs in a staging arena and their placement equals the scan-major bit
buffer -- with the device's slot of 8 words, and with slots of 1 and 0 words, which send units (all units, for 0) down the overflow
path.  Interleaved scans keep their per-unit offsets.  Golden files, every sampling geometry of tests/jpeg_geometry.py, the
coefficient patterns at the run-length and magnitude edges, EOB runs past EOBRUN_MAX and the 937-correction-bit flush, sequential
and progressive."""
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
SLOT_WORDS = 8          # ENC_SLOT_WORDS of csrc/jpeg_gpuenc.cu


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libgpuenc_fused_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gpuenc_fused_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_host.cpp"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_plan.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-o", so, srcs[0], srcs[1]])
    lib = C.CDLL(so)
    lib.emul_fused_check.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_longlong)]
    return lib


def check(emul, data, slots=(SLOT_WORDS, 1, 0)):
    """-> units that overflowed the device's slot, per script (0 sequential, 1 progressive)"""
    over = {}
    for prog in (0, 1):
        for sw in slots:
            n = C.c_longlong(0)
            assert emul.emul_fused_check(data, len(data), prog, sw, C.byref(n)) == 0, (prog, sw)
            if sw == SLOT_WORDS:
                over[prog] = n.value
    return over


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
def test_golden(emul, golden, name):
    check(emul, golden(name))


@pytest.mark.parametrize("name,w,h", CASES)
def test_sampling_geometries(emul, name, w, h):
    check(emul, G.make_jpeg(w, h, G.GEOMETRIES[name], False))


def test_edge_blocks(L, emul):
    """Empty and all-non-zero blocks, extreme coefficients, zero runs of 15, 16, 31, 32, 47 and 48 ahead of a non-zero
    coefficient (the ZRL edges), refinement blocks whose last newly non-zero coefficient is at 63, and a component of 9 x 7 = 63
    blocks (not a multiple of a warp or a CTA).  The all-non-zero blocks overflow the device's slot in the progressive script's
    single-component scans (the sequential script of three components has one interleaved scan)."""
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
    blocks[n, 0] = -32768; blocks[n + 1, 0] = 32767; n += 2
    blocks[n, 63] = 1; blocks[n, 5] = 3; n += 1
    blocks[n, 63] = -1; blocks[n, 1:63] = 2; n += 1
    blocks[n, 1:] = -32767; n += 1
    blocks[n, 1:] = 1; n += 1
    mix = rng.random((len(blocks) - n, 64))
    blocks[n:, 1:] = np.where(mix[:, 1:] < 0.2, rng.integers(-9, 10, size=mix[:, 1:].shape), 0)
    for prog in (1, 0):
        over = check(emul, L.jpeg_encode_coefficients(lay, co, prog))
        assert over[1] > 0, over


@pytest.mark.parametrize("ncomp", [1, 3])
def test_eobrun_max_and_correction_flush(L, emul, ncomp):
    """A component of 257 x 128 = 32,896 blocks: the first 200 blocks hold only AC values of magnitude 2 and 3, so the refinement
    scan buffers 63 correction bits per block with no new coefficient and flushes its EOB run past 937 bits; the remaining blocks
    have no AC coefficient, so each AC scan ends in an EOB run longer than EOBRUN_MAX = 32,767 blocks."""
    lay = _layout(L, 257 * 8, 128 * 8, ncomp)
    co = np.zeros(lay.total_coefs, dtype=np.int16)
    blocks = co.reshape(-1, 64)
    rng = np.random.default_rng(11)
    blocks[:, 0] = rng.integers(-500, 500, size=len(blocks))
    nb = lay.bw[0] * lay.bh[0]
    for c in range(ncomp):
        first = c * nb
        blocks[first:first + 200, 1:] = rng.choice([-3, -2, 2, 3], size=(200, 63))
    check(emul, L.jpeg_encode_coefficients(lay, co, 1), slots=(SLOT_WORDS, 1))
