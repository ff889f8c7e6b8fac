"""Adam7-interlaced PNG input (include/b200_caesium_png_interlaced.h) without a device: the setter, the C header, today's answers with
the switch off, the checks that come before the device with it on, the host decoder against Pillow on every (colour type, depth) and
every combination of empty passes, and the shared geometry (csrc/png_adam7_core.h) run on the CPU against a restatement."""
import ctypes as C
import io
import os
import re
import subprocess
import zlib

import numpy as np
import pytest

from adam7 import SHAPES, adam7_case, adam7_filtered, adam7_pair, layout, pairs, pass_rows, zero_padding
from png_webp_cases import CHANNELS, row_bytes, samples
from pngutil import chunk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caesium-clt_b200")
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
MSG = "interlaced PNG is not supported on the GPU path [3]"


@pytest.fixture
def switch(L):
    yield L.set_png_interlaced
    L.set_png_interlaced(0)


@pytest.fixture
def leg_switches(L):
    """the opt-in legs an Adam7 file can reach, on for the test and back to their defaults afterwards"""
    L.set_png_lossy(1); L.set_png_resize(1); L.set_webp_lossless_convert(1)
    yield
    L.set_png_lossy(0); L.set_png_resize(0); L.set_webp_lossless_convert(0)


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def _legs(L):
    """(name, call) for every leg that takes a PNG source"""
    def params(**kw):
        p = L.default_params()
        for k, v in kw.items():
            setattr(p, k, v)
        return p
    return [
        ("lossless", lambda d: L.compress_in_memory(d, params())),
        ("lossy", lambda d: L.compress_in_memory(d, params(png_optimize=0, png_quality=80))),
        ("resize", lambda d: L.compress_in_memory(d, params(width=3))),
        ("to_size", lambda d: L.compress_to_size_in_memory(d, params(png_optimize=0), 100)),
        ("webp_lossless", lambda d: L.convert_in_memory(d, params(webp_lossless=1), L.FMT_WEBP)),
        ("webp_lossy", lambda d: L.convert_in_memory(d, params(), L.FMT_WEBP)),
        ("jpeg", lambda d: L.convert_in_memory(d, params(), L.FMT_JPEG)),
        ("resize_samples", lambda d: L.png_resize_samples(d, 3, 0)),
        ("decode", lambda d: L.png_decode(d)),
        ("decode_reduced", lambda d: L.png_decode_reduced(d)),
    ]


def _answer(call, data):
    with pytest.raises(Exception) as e:
        call(data)
    return getattr(e.value, "code", None), str(e.value)


def test_setter_accepts_0_and_1_only(L, switch):
    assert switch(0) == 0 and switch(1) == 0
    for bad in (2, -1, 255):
        assert switch(bad) == L.ERR_INVALID_ARGUMENT


def test_header_is_c99_and_links(L, tmp_path):
    exe = str(tmp_path / "c_abi_png_interlaced_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_png_interlaced_check.c"), "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "png interlaced c-abi ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_png_interlaced.h")).read()
    declared = set(re.findall(r"^[a-z_0-9 ]+\b(b200_[a-z0-9_]+)\(", hdr, re.M))
    src = open(os.path.join(ROOT, "tests", "c_abi_png_interlaced_check.c")).read()
    assert declared == {"b200_set_png_interlaced"} and all("(fn)" + f in src for f in declared)


def test_switch_off_every_leg_answers_code_3(L, switch, leg_switches):
    switch(0)
    data = adam7_case(9, 9, 6, 8, seed=1)[0]
    for name, call in _legs(L):
        assert _answer(call, data) == (3, MSG), name
    res = L.compress_batch([data, data], L.default_params())
    assert [(r[1], r[2]) for r in res] == [(3, MSG)] * 2


def _with_interlace_byte(data, method):
    ihdr = bytearray(data[16:29]); ihdr[12] = method
    return data[:8] + chunk(b"IHDR", bytes(ihdr)) + data[33:]


@pytest.mark.parametrize("on", [0, 1])
def test_other_interlace_methods_keep_todays_answer(L, switch, leg_switches, on):
    switch(on)
    inter = adam7_case(9, 9, 2, 8, seed=2)[0]
    for method in (2, 7, 255):
        data = _with_interlace_byte(inter, method)
        for name, call in _legs(L):
            assert _answer(call, data) == (3, MSG), (name, method)


def test_switch_on_checks_before_the_device(L, switch, leg_switches):
    switch(1)
    w, h, ct, bd = 13, 11, 2, 8
    raw = np.random.default_rng(3).integers(0, 256, (h, row_bytes(w, ct, bd)), dtype=np.uint8)
    stream = adam7_filtered(raw, w, h, ct, bd, seed=3)
    ihdr = chunk(b"IHDR", w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([bd, ct, 0, 0, 1]))
    short = b"\x89PNG\r\n\x1a\n" + ihdr + chunk(b"IDAT", zlib.compress(stream[:-30])) + chunk(b"IEND", b"")
    for call in (L.png_decode, L.png_decode_reduced):
        assert _answer(call, short)[0] == 4
    if not _no_gpu():
        pytest.skip("a GPU is visible")
    good = adam7_case(w, h, ct, bd, seed=3)[0]
    for name, call in _legs(L):
        if name.startswith("decode"):
            continue
        assert _answer(call, good)[0] == L.ERR_NO_DEVICE, name


def _pillow_samples(data, ct, bd):
    from PIL import Image
    im = Image.open(io.BytesIO(data)); im.load()
    a = np.asarray(im.convert("L") if im.mode == "1" else im)
    return a.reshape(a.shape[0], a.shape[1], -1).astype(np.int64)


SIZES = SHAPES + [(k, 3) for k in range(1, 18)]


@pytest.mark.parametrize("ct,bd", pairs(), ids=lambda v: str(v))
def test_host_decode_every_pair(L, switch, ct, bd):
    switch(1)
    shapes = SIZES if bd == 1 else SHAPES
    for w, h in shapes:
        for trns in (None, "key" if ct in (0, 2) else "partial" if ct == 3 else None):
            inter, twin, raw, plte, t = adam7_case(w, h, ct, bd, seed=w * 41 + h * 3 + ct + bd, trns=trns)
            info, got = L.png_decode(inter)
            assert (info.width, info.height, info.color_type, info.bit_depth) == (w, h, ct, bd)
            assert np.array_equal(got, raw), (w, h)
            assert np.array_equal(L.png_decode(twin)[1], got)
            if bd == 16:
                continue
            s = samples(got, w, ct, bd)
            if ct == 0 and bd < 8:
                s = s * 255 // ((1 << bd) - 1)
            assert np.array_equal(_pillow_samples(inter, ct, bd), s), (w, h)


def test_host_decode_reduced_equals_the_twin(L, switch):
    switch(1)
    from pngutil import synth
    img = synth(37, 29, 3, seed=5, kind="flat")
    inter, twin = adam7_pair(img.reshape(37, -1), 29, 37, 2, 8, seed=5)
    a, b = L.png_decode_reduced(inter), L.png_decode_reduced(twin)
    assert a[0].color_type == b[0].color_type == 3 and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


# ---- the shared geometry on the CPU ----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libadam7_emul.so")
    srcs = [os.path.join(EMUL_DIR, "adam7_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "png_adam7_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-Werror", "-fPIC", "-shared", "-o", so, srcs[0]])
    return C.CDLL(so)


@pytest.mark.parametrize("ct,bd", pairs(), ids=lambda v: str(v))
def test_core_geometry_and_gather(emul, ct, bd):
    bits = CHANNELS[ct] * bd
    for w, h in SIZES + [(1023, 769)]:
        got = np.zeros(37, np.uint64)
        emul.emul_adam7_layout(C.c_uint32(w), C.c_uint32(h), bits, got.ctypes.data_as(C.c_void_p))
        passes, fo, ro = layout(w, h, bits)
        assert [tuple(int(v) for v in got[5 * p:5 * p + 5]) for p in range(7)] == passes, (w, h)
        assert (int(got[35]), int(got[36])) == (fo, ro)
        raw = zero_padding(np.random.default_rng(w + h).integers(0, 256, (h, row_bytes(w, ct, bd)), dtype=np.uint8), w, ct, bd)
        rows = pass_rows(raw, w, h, ct, bd)
        assert [r.shape for r in rows] == [(ph, rb) if ph else (0, 0) for pw, ph, rb, _, _ in passes]
        packed = np.frombuffer(b"".join(r.tobytes() for r in rows) + b"\0" * 16, np.uint8).copy()
        assert len(packed) == ro + 16 and len(adam7_filtered(raw, w, h, ct, bd)) == fo
        out = np.zeros_like(raw)
        emul.emul_adam7_gather(packed.ctypes.data_as(C.c_void_p), C.c_uint32(w), C.c_uint32(h), bits, out.ctypes.data_as(C.c_void_p))
        assert np.array_equal(out, raw), (w, h)


def test_writer_uses_every_filter_type():
    """the pass rows' filter types, drawn per row, cover all five, Paeth on 1-byte pixels included"""
    w, h, ct, bd = 33, 17, 0, 8
    raw = np.random.default_rng(0).integers(0, 256, (h, w), dtype=np.uint8)
    stream, seen, pos = adam7_filtered(raw, w, h, ct, bd, seed=0), set(), 0
    for pw, ph, rb, _, _ in layout(w, h, 8)[0]:
        for _ in range(ph):
            seen.add(stream[pos]); pos += rb + 1
    assert seen == {0, 1, 2, 3, 4}
