"""Every answer the C ABI gives before it reaches a device, pinned: compress_in_memory, convert_in_memory for every source and
target pair, compress_to_size_in_memory, and the PNG device stage entry points, over garbage, truncated headers, a JPEG with
fractional sampling, target sizes over each format's limit and valid files (code 5 without a device; the lossless JPEG
transcode runs on the host and succeeds), with every opt-in switch off (s0) and on (s1).  The answers are in
golden/c_abi_answers.txt: a `= code message` line, then the cases that answer it, one per line.  Each leg keeps its own order
of refusals, so a change to any of them shows up here as a moved case."""
import io
import os

import pytest

import jpeg_geometry as G
from pngutil import pil_png, synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "c_abi_answers.txt")
SWITCHES = ("set_png_lossy", "set_gif", "set_png_resize", "set_webp_lossless_convert", "set_png_interlaced")


def _webp(arr, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(arr).save(b, "WEBP", **kw)
    return b.getvalue()


def _inputs(golden):
    jpeg = golden("in_420_base_355x237.jpg")
    png = pil_png(synth(30, 40, 3, seed=1))
    webp = _webp(synth(30, 40, 3, seed=2), quality=80)
    gif = golden("g1_head.gif")
    return {
        "jpeg.garbage": b"\xff\xd8\xff" + b"garbage" * 4,
        "jpeg.truncated": jpeg[:40],
        "jpeg.fractional": G.make_jpeg(67, 45, G.FRACTIONAL, False),
        "jpeg.valid": jpeg,
        "png.garbage": b"\x89PNG\r\n\x1a\n" + b"garbage" * 4,
        "png.truncated": png[:20],
        "png.valid": png,
        "webp.garbage": b"RIFF\x24\x00\x00\x00WEBP" + b"garbage" * 4,
        "webp.truncated": webp[:24],
        "webp.valid": webp,
        "webp.alpha": _webp(synth(30, 40, 4, seed=4), quality=80),
        "gif.garbage": b"GIF89a" + b"garbage" * 4,
        "gif.truncated": gif[:20],
        "gif.valid": gif,
        "tiff.garbage": b"II*\x00" + b"garbage" * 4,
        "unknown.garbage": b"garbage" * 4,
    }


# parameter sets: over_webp is above WebP's 16383 only, over_all above every format's limit
PARAMS = {
    "default": {},
    "png_lossless": {"png_optimize": 1},
    "lossless": {"jpeg_optimize": 1, "png_optimize": 1, "webp_lossless": 1},
    "resize": {"width": 24, "png_optimize": 1},
    "resize_lossy": {"width": 24},
    "over_webp": {"width": 20000, "png_optimize": 1},
    "over_all": {"height": 70000},
}
TARGETS = {"jpeg": 0, "png": 1, "gif": 2, "webp": 3}


def _params(L, name):
    p = L.default_params()
    for k, v in PARAMS[name].items():
        setattr(p, k, v)
    return p


def _answer(fn):
    try:
        fn()
    except Exception as e:          # B200Error: code and the message with its " [code]" suffix
        # code 5 carries the CUDA runtime's reason, which depends on the machine
        return (e.code, "no CUDA device") if e.code == 5 else (e.code, str(e))
    return 0, "ok"


def answers(L, golden):
    """case -> (code, message) over every case, with the switches as each case names them"""
    inputs = _inputs(golden)
    out = {}
    for on in (0, 1):
        for s in SWITCHES:
            getattr(L, s)(on)
        try:
            for iname, data in inputs.items():
                for pname in PARAMS:
                    key = f"s{on} {iname} {pname}"
                    out[f"compress {key}"] = _answer(lambda: L.compress_in_memory(data, _params(L, pname)))
                    for tname, fmt in TARGETS.items():
                        out[f"convert->{tname} {key}"] = _answer(lambda: L.convert_in_memory(data, _params(L, pname), fmt))
                    if iname.split(".")[0] in ("jpeg", "png", "webp"):
                        out[f"to_size {key}"] = _answer(lambda: L.compress_to_size_in_memory(data, _params(L, pname), len(data) // 2))
                if iname.startswith("png."):
                    out[f"png_device_times s{on} {iname}"] = _answer(lambda: L.png_device_times(data))
                    for w in (0, 24, 70000):
                        out[f"png_resize_samples s{on} {iname} width={w}"] = _answer(lambda: L.png_resize_samples(data, w, 0))
        finally:
            for s in SWITCHES:
                getattr(L, s)(0)
    return out


def _read_golden():
    pinned, answer = {}, None
    with open(GOLDEN, encoding="utf-8") as f:
        for line in f.read().splitlines():
            if line.startswith("= "):
                code, msg = line[2:].split(" ", 1)
                answer = (int(code), msg)
            else:
                pinned[line] = answer
    return pinned


def test_answers_before_the_device_are_pinned(L, golden):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    got = answers(L, golden)
    pinned = _read_golden()
    assert sorted(got) == sorted(pinned)
    changed = [(case, pinned[case], got[case]) for case in pinned if got[case] != pinned[case]]
    assert not changed, changed[:20]
