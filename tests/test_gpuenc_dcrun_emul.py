"""CPU checks of the device encoder's DC-first interleaved scan (tests/emul/gpuenc_dcrun_emul.cpp): one thread per MCU codes the
MCU's units from the compact DC array into a slot, a CTA's MCUs make one run in a staging arena, and the runs are placed into the
scan; run CTA by CTA, the result equals the scan coded unit after unit, bit for bit.  Every sampling geometry of
tests/jpeg_geometry.py at MCU counts that are not multiples of the CTA size, decoded DC values and DC values whose differences are
all of category 11 (also against the predictor 0 at each component's start), CTAs of the kernel's 128 MCUs and of 32 and 5, and
slots of the kernel's 8 words, 1 word and none (every MCU, the 10-block ones included, down the overflow path)."""
import ctypes as C
import os
import subprocess

import pytest

import jpeg_geometry as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
CTA = 128               # ENC_DC_MCUS of csrc/jpeg_gpuenc_plan.h
SLOT_WORDS = 8          # ENC_SLOT_WORDS of csrc/jpeg_gpuenc.cu
COLOUR = {name: f for name, f in G.GEOMETRIES.items() if len(f) > 1}
CASES = [(name, w, h) for name, f in COLOUR.items() for (w, h) in G.sizes_for(f)]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libgpuenc_dcrun_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gpuenc_dcrun_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_host.cpp"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_plan.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-o", so, srcs[0], srcs[1]])
    lib = C.CDLL(so)
    lib.emul_dcrun_check.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong)]
    return lib


def check(emul, data, dc_mode, cta, slot_words):
    n = C.c_longlong(0)
    assert emul.emul_dcrun_check(data, len(data), dc_mode, cta, slot_words, C.byref(n)) == 0, (dc_mode, cta, slot_words)
    return n.value


@pytest.mark.parametrize("name,w,h", CASES)
def test_sampling_geometries(emul, name, w, h):
    data = G.make_jpeg(w, h, COLOUR[name], False)
    for dc_mode in (0, 1, 2):
        for cta in (CTA, 32, 5):
            for sw in (SLOT_WORDS, 1, 0):
                over = check(emul, data, dc_mode, cta, sw)
                if sw == 0:
                    assert over > 0
    if G.mcu_blocks(COLOUR[name]) == 10:        # 10 units of a category-11 difference: more than one slot word
        assert check(emul, data, 1, CTA, 1) > 0


def test_golden_progressive(emul, golden):
    for name in ("in_420_prog_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg", "in_420_tiny_3x3.jpg"):
        for dc_mode in (0, 1):
            check(emul, golden(name), dc_mode, CTA, SLOT_WORDS)


def test_grey_has_no_interleaved_scan(emul, golden):
    data = golden("in_gray_base_355x237.jpg")
    assert emul.emul_dcrun_check(data, len(data), 0, CTA, SLOT_WORDS, None) == 3
