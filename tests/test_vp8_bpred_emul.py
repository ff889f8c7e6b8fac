"""k_vp8_encode_bpred as the device runs it (csrc/vp8_kernels.cu, emulated serially by tests/emul/vp8_bpred_emul.cpp through
csrc/vp8_bpred_core.h: the trail-by-two wavefront with every cross-macroblock read checked against the macroblocks already finished,
phase A's lane layout and reductions, the 10 anti-diagonal steps with lane 10 s + m on mode m of the step's s-th block, the scan of
the scores with ties to the lower mode) equals the scalar twin (oracle/webp_bpred_oracle.c), which codes sub-blocks in raster
order: the same levels, modes, sub-block modes and reconstruction.  The shapes include one-macroblock-wide and one-row frames (the
frame's top row and last column on every macroblock) and the last column of wider frames."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from pngutil import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
CSRC = os.path.join(ROOT, "caesium-clt_b200", "csrc")


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libvp8_bpred_emul.so")
    srcs = [os.path.join(EMUL_DIR, "vp8_bpred_emul.cpp"), os.path.join(CSRC, "vp8_bpred_core.h"), os.path.join(CSRC, "vp8_tables.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, srcs[0]])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def OB(O):
    from oracle import webp_bpred
    return webp_bpred


def run(emul, O, rgb, q):
    _, h, w = rgb.shape
    mbw, mbh = (w + 15) // 16, (h + 15) // 16
    nmb = mbw * mbh
    Y, U, V = O.webp_rgb_to_yuv(rgb)
    f = np.array(O.vp8_quant_factors(O.vp8_qindex(q)), np.int32)
    levels = np.zeros((nmb, 25, 16), np.int16); modes = np.zeros((nmb, 4), np.uint8); bmodes = np.zeros((nmb, 16), np.uint8)
    RY, RU, RV = np.zeros_like(Y), np.zeros_like(U), np.zeros_like(V)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    bad = emul.emul_vp8_bpred(p(Y), p(U), p(V), mbw, mbh, p(f), p(levels), p(modes), p(bmodes), p(RY), p(RU), p(RV))
    return bad, levels, modes, bmodes, RY, RU, RV


@pytest.mark.parametrize("h,w,q,kind", [(64, 64, 75, "photo"), (37, 53, 50, "photo"), (1, 1, 80, "flat"), (300, 16, 60, "photo"),
                                        (16, 300, 40, "noise"), (129, 65, 85, "noise"), (96, 160, 30, "flat"), (200, 300, 100, "photo"),
                                        (33, 17, 0, "photo"), (48, 250, 90, "noise")])
def test_kernel_decomposition_equals_the_twin(emul, O, OB, h, w, q, kind):
    rgb = np.ascontiguousarray(synth(h, w, 3, seed=h + w + q, kind=kind).transpose(2, 0, 1))
    bad, levels, modes, bmodes, RY, RU, RV = run(emul, O, rgb, q)
    st = OB.webp_bpred_stages(rgb, q)
    assert bad == 0, "a macroblock read output the trail-by-two wavefront had not finished"
    assert np.array_equal(modes, st["modes"]) and np.array_equal(bmodes, st["bmodes"])
    assert np.array_equal(levels, st["levels"])
    assert np.array_equal(RY, st["Yraw"]) and np.array_equal(RU, st["U"]) and np.array_equal(RV, st["V"])


def test_cases_take_both_arms(emul, O):
    rgb = np.ascontiguousarray(synth(96, 160, 3, seed=3, kind="photo").transpose(2, 0, 1))
    _, _, modes, bmodes, *_ = run(emul, O, rgb, 60)
    assert (modes[:, 0] == 4).any() and (modes[:, 0] != 4).any() and len(np.unique(bmodes[modes[:, 0] == 4])) >= 8
