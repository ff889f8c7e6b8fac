"""The growth rules of dev_buffer.h against the formulas each owner allocated by before the rules moved there.  Slots only grow, so
the rules fix the library's device-memory footprint; a changed rule changes how many PNG callers fit on one card."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
KIB64 = 1 << 16


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libdev_buffer_emul.so")
    srcs = [os.path.join(EMUL_DIR, "dev_buffer_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "dev_buffer.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-fPIC", "-shared", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emul_grow_bytes.argtypes = [C.c_char_p, C.c_void_p, C.c_void_p, C.c_size_t]
    return lib


def pow2_at_least(want):
    """the smallest power of two that is >= 64 KiB and >= want"""
    return max(KIB64, 1 << max(0, want - 1).bit_length())


# owner -> (rule name in dev_buffer.h, the size it allocates for a request of `need` bytes)
RULES = {
    "Slot (JPEG coefficients, scratch, parameter block)": ("slot", lambda need: -(-(need + need // 8) // KIB64) * KIB64),
    "GpuEncoder / GpuDecoder": ("pow2_half", lambda need: pow2_at_least(need + need // 2)),
    "PngDevice / PngQuant growable buffers": ("pow2_quarter", lambda need: pow2_at_least(need + need // 4)),
    "WebpDevice / Vp8lDevice": ("pow2", lambda need: pow2_at_least(need)),
    "PngQuant fixed buffers, PNG stage helpers": ("exact", lambda need: need),
}


def sizes():
    s = {0, 1, KIB64 - 1, KIB64, KIB64 + 1}
    for k in range(37):
        s.update({(1 << k) - 1, 1 << k, (1 << k) + 1})
    rng = np.random.default_rng(2024)
    s.update(int(v) for v in rng.integers(0, 1 << 36, 3000, dtype=np.int64))
    s.update(int(v) for v in rng.integers(0, 1 << 22, 1000, dtype=np.int64))
    return sorted(s)


@pytest.mark.parametrize("owner", sorted(RULES))
def test_rule_matches_the_owner_formula(emul, owner):
    rule, formula = RULES[owner]
    need = np.array(sizes(), dtype=np.uint64)
    got = np.zeros_like(need)
    assert emul.emul_grow_bytes(rule.encode(), need.ctypes.data, got.ctypes.data, need.size) == 0
    want = np.array([formula(int(n)) for n in need], dtype=np.uint64)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(int(need[i]), int(got[i]), int(want[i])) for i in bad[:5]]
    assert (got >= need).all()

