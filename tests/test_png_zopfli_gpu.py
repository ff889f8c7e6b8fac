"""PNG `--zopfli` on the device (b200_set_png_zopfli + png_force_zopfli): the device parse equals the twin token for token, and every
PNG output keeps its filter choice, is never larger than without the flag, and carries the smaller of the default payload and the
host writer's coding of the twin's tokens (the default on a tie)."""
import io
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import png_zopfli_cases as cases
from adam7 import adam7_case
from png_webp_cases import DEPTHS, make_case
from pngutil import idat_stream, pil_png

from oracle import png_zopfli as Z

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def switches(L):
    L.set_png_lossy(1); L.set_png_resize(1); L.set_png_interlaced(1)
    yield
    L.set_png_zopfli(0); L.set_png_lossy(0); L.set_png_resize(0); L.set_png_interlaced(0)


def _params(L, **kw):
    """lossless (png_optimize = 1) unless kw says otherwise"""
    p = L.default_params()
    p.png_optimize = 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


# ---- the parse ---------------------------------------------------------------------------------------------------------------
def _streams():
    out = [(f"{name}_s{s}", *cases.filtered(img, s)) for name, img in cases.images().items() for s in (0, 4)]
    out += [(f"n{n}", *cases.boundary_stream(n)) for n in (1, 2, 3, cases.SEG - 1, cases.SEG, cases.SEG + 1)]
    return out


@pytest.mark.parametrize("case", _streams(), ids=lambda c: c[0])
def test_device_parse_equals_the_twin(L, case):
    _, st, bpp, stride = case
    for b in sorted({bpp, 1, 2, 4, 6, 8}):        # the filter distance only moves the fixed candidates: every bpp on every stream
        assert np.array_equal(L.png_lz77_zopfli(st, b, stride), Z.lz77_zopfli(st, b, stride)), b
    s16 = cases.filtered(np.ascontiguousarray(cases.photo(30, 20)[:, :, :2]).view(np.uint8))[0]
    assert np.array_equal(L.png_lz77_zopfli(s16, 2, 61), Z.lz77_zopfli(s16, 2, 61))


@pytest.mark.parametrize("n", [cases.SLICE - 1, cases.SLICE + 1])
def test_device_parse_equals_the_twin_at_the_slice_edge(L, n):
    st, bpp, stride = cases.boundary_stream(n)
    assert np.array_equal(L.png_lz77_zopfli(st, bpp, stride), Z.lz77_zopfli(st, bpp, stride))


# ---- whole files -----------------------------------------------------------------------------------------------------------
def _filtered_and_payload(png):
    (w, h, bd, ct, _, _, _), idat, _ = idat_stream(png)
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ct]
    bits = bd * ch
    return zlib.decompress(idat), idat, max(1, bits // 8), (w * bits + 7) // 8 + 1


def _pixels(png):
    from PIL import Image
    im = Image.open(io.BytesIO(png)); im.load()
    return np.asarray(im.convert("RGBA") if im.mode not in ("I", "I;16", "I;16B") else im)


def _check_pair(L, off, on):
    """the same filtered stream and pixels, no larger, and the payload is min(off, the twin's tokens coded by the host writer)"""
    f_off, z_off, bpp, stride = _filtered_and_payload(off)
    f_on, z_on, _, _ = _filtered_and_payload(on)
    assert f_on == f_off
    assert np.array_equal(_pixels(on), _pixels(off))
    assert len(on) <= len(off)
    st = np.frombuffer(f_off, np.uint8)
    z_twin = L.png_deflate_tokens(Z.lz77_zopfli(st, bpp, stride), zlib.adler32(f_off))
    assert z_on == (z_twin if len(z_twin) < len(z_off) else z_off)
    assert off[:33] == on[:33]


def _file_cases():
    out = []
    for ct, depths in DEPTHS.items():
        for bd in depths:
            for trns in ([None, "key"] if ct in (0, 2) else [None, "partial"] if ct == 3 else [None]):
                out.append((f"ct{ct}_bd{bd}_{trns or 'plain'}", make_case(37, 23, ct, bd, seed=bd + ct, trns=trns)[0]))
    out.append(("flat_rgb", pil_png(cases.flat(160, 96))))
    out.append(("text_rgb", pil_png(cases.text(200, 64))))
    out.append(("photo_rgba", pil_png(np.dstack([cases.photo(96, 64), np.full((64, 96), 200, np.uint8)]))))
    out.append(("palette_reducible", pil_png(np.repeat(np.repeat(cases.flat(24, 16), 4, 0), 4, 1))))
    out.append(("adam7", adam7_case(41, 29, 6, 8, seed=3)[0]))
    return out


@pytest.mark.parametrize("case", _file_cases(), ids=lambda c: c[0])
def test_lossless_files(L, case):
    _, data = case
    L.set_png_zopfli(1)
    off = L.compress_in_memory(data, _params(L))
    on = L.compress_in_memory(data, _params(L, png_force_zopfli=1))
    _check_pair(L, off, on)


@pytest.mark.parametrize("level", range(7))
def test_every_level(L, level):
    data = pil_png(cases.text(120, 48))
    L.set_png_zopfli(1)
    _check_pair(L, L.compress_in_memory(data, _params(L, png_optimization_level=level)),
                L.compress_in_memory(data, _params(L, png_optimization_level=level, png_force_zopfli=1)))


def test_lossy_resize_jpeg_and_to_size(L):
    flat = pil_png(cases.flat(160, 96))
    from tools.synth import synth_jpeg
    jpg = synth_jpeg(96, 64)
    L.set_png_zopfli(1)
    for kw in ({"png_optimize": 0, "png_quality": 60}, {"width": 80}):
        _check_pair(L, L.compress_in_memory(flat, _params(L, **kw)), L.compress_in_memory(flat, _params(L, png_force_zopfli=1, **kw)))
    _check_pair(L, L.convert_in_memory(jpg, _params(L), L.FMT_PNG), L.convert_in_memory(jpg, _params(L, png_force_zopfli=1), L.FMT_PNG))
    off = L.compress_to_size_in_memory(flat, _params(L, png_optimize=0), 2500)
    on = L.compress_to_size_in_memory(flat, _params(L, png_optimize=0, png_force_zopfli=1), 2500)
    assert len(on) <= 2500 or len(on) <= len(off)
    assert zlib.decompress(idat_stream(on)[1]) and _pixels(on).shape == _pixels(off).shape


def test_switch_and_flag_each_alone_change_nothing(L):
    data = pil_png(cases.text(200, 64))
    L.set_png_zopfli(0)
    base = L.compress_in_memory(data, _params(L))
    assert L.compress_in_memory(data, _params(L, png_force_zopfli=1)) == base
    L.set_png_zopfli(1)
    assert L.compress_in_memory(data, _params(L)) == base
    assert len(L.compress_in_memory(data, _params(L, png_force_zopfli=1))) < len(base)


def test_environment_variable_turns_the_switch_on_once(tmp_path):
    import os
    import subprocess
    import sys
    code = ("import os, sys; sys.path.insert(0, sys.argv[1]); import __graft_entry__ as g; L = g._pkg(); "
            "sys.path.insert(0, os.path.join(sys.argv[1], 'tests')); import png_zopfli_cases as c; from pngutil import pil_png; "
            "d = pil_png(c.text(200, 64)); p = L.default_params(); p.png_optimize = 1; p.png_force_zopfli = 1; a = L.compress_in_memory(d, p); "
            "os.environ['B200_PNG_ZOPFLI'] = 'off'; b = L.compress_in_memory(d, p); L.set_png_zopfli(0); "
            "c0 = L.compress_in_memory(d, p); print(len(a), len(b), len(c0), a == b, c0 != a)")
    r = subprocess.run([sys.executable, "-c", code, cases.ROOT], capture_output=True, text=True, env=dict(os.environ, B200_PNG_ZOPFLI="gpu"))
    assert r.returncode == 0, r.stderr
    assert r.stdout.split()[-2:] == ["True", "True"], r.stdout


def test_batch_and_threads_equal_single_calls(L):
    L.set_png_zopfli(1)
    datas = [pil_png(cases.text(120 + 8 * k, 40)) for k in range(4)] + [pil_png(cases.flat(100, 60, k)) for k in range(4)]
    p = _params(L, png_force_zopfli=1)
    single = [L.compress_in_memory(d, p) for d in datas]
    assert [r[0] for r in L.compress_batch(datas, p)] == single
    with ThreadPoolExecutor(8) as ex:
        assert list(ex.map(lambda d: L.compress_in_memory(d, p), datas)) == single


@pytest.mark.parametrize("name", ["photo_4096_rgba", "flat_3840x2160"])
def test_large_images_finish_and_round_trip(L, name):
    if name.startswith("photo"):
        img = np.dstack([cases.photo(4096, 4096), np.full((4096, 4096), 255, np.uint8)])
        img[::3, ::5, 3] = 128
    else:
        img = cases.flat(3840, 2160)
    data = pil_png(img, compress_level=1)
    L.set_png_zopfli(1)
    off = L.compress_in_memory(data, _params(L))
    t = time.perf_counter()
    on = L.compress_in_memory(data, _params(L, png_force_zopfli=1))
    dt = time.perf_counter() - t
    assert len(on) <= len(off)
    assert zlib.decompress(idat_stream(on)[1]) == zlib.decompress(idat_stream(off)[1])
    assert np.array_equal(_pixels(on), _pixels(off))
    print(f"{name}: {len(off)} -> {len(on)} bytes, {dt * 1e3:.0f} ms with --zopfli")
