"""Conversions to and from GIF without a device (include/b200_caesium_gif_convert.h): the switch and its environment variable, the C
header, today's answers with the switch off, the frame-0 decoder against a numpy restatement on gifutil's parser, its handling of
damage before and after frame 0, and the canvas rule of converted sources."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import gif_cases
import gifutil
from gif_convert_cases import canvas, first_frame, sources, twin
from pngutil import pil_png, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "caesium-clt_b200")
FMT_JPEG, FMT_PNG, FMT_GIF, FMT_WEBP = 0, 1, 2, 3
OUTSIDE = "this conversion is outside the GPU path (route to caesium::convert_in_memory) [3]"
FROM_OUTSIDE = "conversion from this format is outside the GPU path (route to caesium::convert_in_memory) [3]"


@pytest.fixture
def switch(L):
    yield L.set_gif_convert
    L.set_gif_convert(0)


def _code(L, data, p, fmt):
    with pytest.raises(L.B200Error) as e:
        L.convert_in_memory(data, p, fmt)
    return e.value.code, str(e.value)


def _webp():
    import io
    from PIL import Image
    b = io.BytesIO(); Image.fromarray(synth(20, 30, 3, seed=3)).save(b, "WEBP", quality=80)
    return b.getvalue()


def test_setter_accepts_0_and_1_only(L, switch):
    assert switch(0) == 0 and switch(1) == 0
    assert switch(2) == L.ERR_INVALID_ARGUMENT and switch(-1) == L.ERR_INVALID_ARGUMENT


def test_header_is_c99_and_links(L, tmp_path):
    exe = str(tmp_path / "c_abi_gif_convert_check")
    cmd = ["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c_abi_gif_convert_check.c"), "-o", exe, "-L", PKG, "-lb200caesium", "-Wl,-rpath," + PKG]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "gif convert c-abi ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
    hdr = open(os.path.join(ROOT, "include", "b200_caesium_gif_convert.h")).read()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", hdr)) - {"b200_status"}
    src = open(os.path.join(ROOT, "tests", "c_abi_gif_convert_check.c")).read()
    assert declared == {"b200_set_gif_convert", "b200_gif_first_frame"} and all("(fn)" + f in src for f in declared)


def test_switch_off_answers_are_unchanged(L, golden, switch):
    """every route answers code 3 with the message of the library before the conversions existed, also with the GIF leg on"""
    switch(0)
    gif = dict(gif_cases.cases())["anim_disposal1"]
    try:
        for gif_leg in (0, 1):
            L.set_gif(gif_leg)
            for data, fmt, msg in ((golden("in_420_base_355x237.jpg"), FMT_GIF, OUTSIDE), (pil_png(synth(20, 30, 3, seed=1)), FMT_GIF, OUTSIDE),
                                   (_webp(), FMT_GIF, OUTSIDE), (gif, FMT_JPEG, OUTSIDE), (gif, FMT_PNG, OUTSIDE), (gif, FMT_WEBP, FROM_OUTSIDE),
                                   (gif[:40], FMT_PNG, OUTSIDE), (b"garbage", FMT_GIF, "Unknown file type [2]"), (gif, FMT_GIF, "Cannot convert to the same format [8]")):
                assert _code(L, data, L.default_params(), fmt) == (int(msg[-2]), msg)
    finally:
        L.set_gif(0)


_ENV_SCRIPT = r"""
import os, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import conftest
conftest._import_pkg()
import caesium_clt_b200._lib as L
import gif_cases
bad = dict(gif_cases.cases())["anim_disposal1"][:60]          # cut before frame 0 ends: code 4 when the route is taken, else code 3
def code():
    try:
        L.convert_in_memory(bad, L.default_params(), L.FMT_JPEG)
    except L.B200Error as e:
        return e.code
codes = [code()]
os.environ["B200_GIF_CONVERT"] = "off" if codes[0] == 4 else "gpu"     # read once: a later change is not seen
codes.append(code())
L.set_gif_convert(1); codes.append(code())
L.set_gif_convert(0); codes.append(code())
print(codes)
"""


@pytest.mark.parametrize("env,want", [(None, [3, 3, 4, 3]), ("gpu", [4, 4, 4, 3]), ("on", [3, 3, 4, 3])])
def test_environment_is_read_once(env, want):
    e = {k: v for k, v in os.environ.items() if k != "B200_GIF_CONVERT"}
    if env is not None:
        e["B200_GIF_CONVERT"] = env
    r = subprocess.run([sys.executable, "-c", _ENV_SCRIPT.format(root=ROOT)], capture_output=True, text=True, env=e)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == str(want)


@pytest.mark.parametrize("name,data", sources(), ids=[n for n, _ in sources()])
def test_first_frame_equals_restatement(L, name, data):
    got = L.gif_first_frame(data)
    want = first_frame(data)
    assert got.shape == want.shape and np.array_equal(got, want), name


def test_first_frame_keeps_the_transparent_colour(L):
    idx = np.array([[0, 1, 1], [2, 1, 0]], np.uint8)
    data = gif_cases.raw_gif(5, 4, [dict(x=1, y=2, idx=idx, transparent=1, table=[(9, 8, 7), (200, 100, 50), (1, 2, 3), (0, 0, 0)], m=2)])
    got = L.gif_first_frame(data)
    assert (got[:2] == 0).all() and (got[:, :1] == 0).all() and (got[:, 4:] == 0).all()
    assert got[2, 2].tolist() == [200, 100, 50, 0] and got[3, 2].tolist() == [200, 100, 50, 0] and got[2, 1].tolist() == [9, 8, 7, 255]
    # the composited canvas of the re-encoder clears the same pixel
    assert gifutil.decode(data)[0][0][0][2, 2].tolist() == [0, 0, 0, 0]


def _two_frames(second):
    rng = np.random.default_rng(3)
    f0 = dict(x=2, y=1, idx=rng.integers(0, 8, (6, 9)).astype(np.uint8), transparent=5, m=3)
    gct = [tuple(int(v) for v in c) for c in rng.integers(0, 256, (8, 3))]
    one = gif_cases.raw_gif(14, 10, [f0], gct=gct)
    return one, gif_cases.raw_gif(14, 10, [f0, second], gct=gct)


def test_damage_after_frame_0_is_not_seen(L):
    one, two = _two_frames(dict(x=0, y=0, idx=np.ones((10, 14), np.uint8)))
    head = one[:-1]                                     # the same bytes up to the end of frame 0's image data
    assert two.startswith(head)
    want = first_frame(one)
    past = gif_cases.raw_gif(14, 10, [dict(x=9, y=0, idx=np.zeros((3, 7), np.uint8))], gct=[(1, 1, 1), (2, 2, 2)])
    for bad in (head, head + b"\x21", two[:len(head) + 30], head + b"\x99junk", head + past[past.index(b"\x2c"):]):
        assert np.array_equal(L.gif_first_frame(bad), want)
        with pytest.raises(L.B200Error) as e:           # the re-encoder reads the whole file and refuses it
            L.gif_decode(bad)
        assert e.value.code in (L.ERR_CORRUPT_INPUT, L.ERR_UNSUPPORTED)


def test_damage_inside_frame_0_is_corrupt(L):
    one, _ = _two_frames(dict(x=0, y=0, idx=np.ones((10, 14), np.uint8)))
    start = one.index(b"\x2c", 13 + 24)                 # the image descriptor after the global table and the GCE
    cases = [one[:k] for k in (start - 3, start + 1, start + 9, start + 11, len(one) - 4)]
    bad_code = bytearray(one); bad_code[start + 12] = 0xFF; cases.append(bytes(bad_code))       # a code past the dictionary
    bad_m = bytearray(one); bad_m[start + 10] = 9; cases.append(bytes(bad_m))                   # minimum code size 9
    cases.append(gif_cases.raw_gif(4, 4, [dict(x=0, y=0, idx=np.zeros((2, 2), np.uint8))]))   # no colour table at all
    cases.append(one[:start] + b"\x3b")                 # a trailer before any frame
    for k, bad in enumerate(cases):
        with pytest.raises(L.B200Error) as e:
            L.gif_first_frame(bad)
        assert e.value.code == L.ERR_CORRUPT_INPUT, k


def test_frame_0_past_the_screen_is_unsupported(L):
    past = gif_cases.raw_gif(6, 2, [dict(x=3, y=0, idx=np.zeros((2, 4), np.uint8), table=[(0, 0, 0), (1, 1, 1)], m=2)])
    with pytest.raises(L.B200Error) as e:
        L.gif_first_frame(past)
    assert e.value.code == L.ERR_UNSUPPORTED


def test_canvas_rule(O):
    """alpha 0 is clear whatever the colour; alpha 1..255 is opaque; the twin's file shows exactly that"""
    rgba = np.zeros((4, 5, 4), np.uint8)
    rgba[..., :3] = np.arange(60, dtype=np.uint8).reshape(4, 5, 3) * 4 + 1
    rgba[..., 3] = np.array([0, 1, 254, 255, 0] * 4).reshape(4, 5)
    c = canvas(rgba)
    assert (c[rgba[..., 3] == 0] == 0).all()
    assert (c[rgba[..., 3] != 0, 3] == 255).all() and np.array_equal(c[rgba[..., 3] != 0, :3], rgba[rgba[..., 3] != 0, :3])
    frames, loop = gifutil.decode(twin(rgba, 100))
    assert loop is None and len(frames) == 1 and frames[0][1] == 0
    assert np.array_equal(frames[0][0], c)              # at quality 100 an image of at most 256 values is kept exactly


def test_switch_on_checks_before_the_device(L, golden, switch):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    switch(1)
    p = L.default_params()
    gif = dict(gif_cases.cases())["anim_disposal1"]
    assert _code(L, golden("in_420_base_355x237.jpg"), p, FMT_GIF)[0] == L.ERR_NO_DEVICE
    assert _code(L, pil_png(synth(20, 30, 3, seed=1)), p, FMT_GIF)[0] == L.ERR_NO_DEVICE
    assert _code(L, _webp(), p, FMT_GIF)[0] == L.ERR_NO_DEVICE
    p.width = 10
    assert _code(L, golden("in_420_base_355x237.jpg"), p, FMT_GIF) == (3, "GIF resize is outside the GPU path (route to caesium::convert_in_memory) [3]")
    p = L.default_params(); p.webp_lossless = 1
    assert _code(L, gif, p, FMT_WEBP)[0] == L.ERR_UNSUPPORTED
    p = L.default_params()
    assert _code(L, gif[:60], p, FMT_JPEG)[0] == L.ERR_CORRUPT_INPUT
    for fmt in (FMT_JPEG, FMT_WEBP):
        assert _code(L, gif, p, fmt)[0] == L.ERR_NO_DEVICE
