"""The PNG-row -> ARGB rule of the lossless WebP conversion (csrc/png_pixel_core.h, run by the device kernels of csrc/png_webp.cu and
here on the CPU by tests/emul/png_pixel_emul.cpp) equals a numpy restatement for every colour type, bit depth and tRNS form."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from png_webp_cases import cases, expected_rgba, make_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libpng_pixel_emul.so")
    srcs = [os.path.join(EMUL_DIR, "png_pixel_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "png_pixel_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-fPIC", "-shared", "-o", so, srcs[0]])
    return C.CDLL(so)


def _run(emul, raw, w, ct, bd, plte, trns):
    raw = np.ascontiguousarray(raw, np.uint8)
    h, rb = raw.shape
    out = np.zeros(h * w, np.uint32)
    pb, tb = (C.c_uint8 * max(1, len(plte))).from_buffer_copy(plte or b"\0"), (C.c_uint8 * max(1, len(trns))).from_buffer_copy(trns or b"\0")
    emul.emul_png_rows_argb(raw.ctypes.data_as(C.c_void_p), C.c_size_t(rb), w, h, ct, bd, pb, C.c_size_t(len(plte)), tb, C.c_size_t(len(trns)),
                            out.ctypes.data_as(C.c_void_p))
    argb = out.reshape(h, w)
    return np.stack([(argb >> 16) & 255, (argb >> 8) & 255, argb & 255, argb >> 24], axis=-1).astype(np.uint8)


@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_rule_equals_the_restatement(emul, case):
    _, w, h, ct, bd, trns, plte_len = case
    _, raw, plte, t = make_case(w, h, ct, bd, seed=w * 31 + h * 7 + ct * 5 + bd, trns=trns, plte_len=plte_len)
    want = expected_rgba(raw, w, ct, bd, plte, t)
    assert np.array_equal(_run(emul, raw, w, ct, bd, plte, t), want)


def test_restatement_hits_every_branch():
    """the cases above exercise what they claim: keys that match, soft palette alphas, indices past PLTE, 16-bit high bytes"""
    data, raw, plte, t = make_case(13, 7, 0, 8, seed=1, trns="key")
    assert (expected_rgba(raw, 13, 0, 8, plte, t)[..., 3] == 0).sum() >= 2
    data, raw, plte, t = make_case(13, 7, 2, 16, seed=2, trns="key")
    assert expected_rgba(raw, 13, 2, 16, plte, t)[0, 0, 3] == 0
    data, raw, plte, t = make_case(13, 7, 3, 8, seed=3, trns="partial", plte_len=200)
    rgba = expected_rgba(raw, 13, 3, 8, plte, t)
    idx = raw[:, :13]
    assert (rgba[idx >= 200][:, :3] == 0).all() and (idx >= 200).any()
    assert set(np.unique(rgba[idx < 4][:, 3])) <= {0, 128, 255, 7}
    s = np.array([[0xAB, 0xCD]], np.uint8)
    assert expected_rgba(s, 1, 0, 16)[0, 0, 0] == 0xAB
