"""The lossless WebP conversion switch (include/b200_caesium_webp_lossless.h) without a device: the setter, the C header, today's
answers with the switch off, and the checks that come before the device with it on."""
import os
import re
import subprocess
import zlib

import pytest

from pngutil import chunk, pil_png, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caesium-clt_b200")


@pytest.fixture
def switch(L):
    yield L.set_webp_lossless_convert
    L.set_webp_lossless_convert(0)


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def _params(L):
    p = L.default_params(); p.webp_lossless = 1
    return p


def _code(L, data, p, fmt):
    with pytest.raises(L.B200Error) as e:
        L.convert_in_memory(data, p, fmt)
    return e.value.code, str(e.value)


def _interlaced():
    ihdr = chunk(b"IHDR", (5).to_bytes(4, "big") + (4).to_bytes(4, "big") + bytes([8, 0, 0, 0, 1]))
    return b"\x89PNG\r\n\x1a\n" + ihdr + chunk(b"IDAT", zlib.compress(bytes(64))) + chunk(b"IEND", b"")


def test_setter_accepts_0_and_1_only(L, switch):
    assert switch(0) == 0 and switch(1) == 0
    assert switch(2) == L.ERR_INVALID_ARGUMENT and switch(-1) == L.ERR_INVALID_ARGUMENT


def test_header_is_c99_and_links(L, tmp_path):
    exe = str(tmp_path / "c_abi_webp_lossless_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_webp_lossless_check.c"), "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "webp lossless c-abi ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_webp_lossless.h")).read()
    declared = set(re.findall(r"^[a-z_0-9 ]+\b(b200_[a-z0-9_]+)\(", hdr, re.M))
    src = open(os.path.join(ROOT, "tests", "c_abi_webp_lossless_check.c")).read()
    assert declared == {"b200_set_webp_lossless_convert"} and all("(fn)" + f in src for f in declared)


def test_switch_off_answers_are_unchanged(L, golden, switch):
    switch(0)
    msg = "lossless WebP (VP8L) is outside the GPU path (route to caesium::convert_in_memory) [3]"
    for data in (golden("in_420_base_355x237.jpg"), pil_png(synth(20, 30, 3, seed=1)), _interlaced(), pil_png(synth(1, 16384, 1))):
        assert _code(L, data, _params(L), L.FMT_WEBP) == (3, msg)


def test_switch_on_checks_before_the_device(L, golden, switch):
    if not _no_gpu():
        pytest.skip("a GPU is visible")
    switch(1)
    p = _params(L)
    assert _code(L, b"garbage", p, L.FMT_WEBP)[0] == L.ERR_UNKNOWN_FORMAT
    assert _code(L, _interlaced(), p, L.FMT_WEBP)[0] == L.ERR_UNSUPPORTED
    code, msg = _code(L, pil_png(synth(1, 16384, 1)), p, L.FMT_WEBP)
    assert code == L.ERR_INVALID_ARGUMENT and msg == "invalid dimensions for WebP [1]"
    assert _code(L, pil_png(synth(20, 30, 3, seed=1)), p, L.FMT_WEBP)[0] == L.ERR_NO_DEVICE
    assert _code(L, golden("in_420_base_355x237.jpg"), p, L.FMT_WEBP)[0] == L.ERR_NO_DEVICE


def test_compress_to_size_stays_refused(L, switch):
    from PIL import Image
    import io
    b = io.BytesIO(); Image.fromarray(synth(40, 50, 3, seed=2)).save(b, "WEBP", lossless=True); src = b.getvalue()
    for on in (0, 1):
        switch(on)
        with pytest.raises(L.B200Error) as e:
            L.compress_to_size_in_memory(src, _params(L), len(src) // 2)
        assert e.value.code == 3
