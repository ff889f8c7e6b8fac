"""Adam7-interlaced PNG input on the device (b200_set_png_interlaced): on every PNG leg an Adam7 file gives the bytes its non-interlaced
twin gives.  The twin's rows take the non-interlaced un-filter, which shares no code with the pass wavefront and the gather, so this
checks the de-interlace on the device (and on the host decoder behind the JPEG and lossy WebP conversions) end to end."""
import io
import zlib

import numpy as np
import pytest

from adam7 import SHAPES, adam7_case, adam7_filtered, adam7_pair, layout, pairs
from png_webp_cases import CHANNELS, row_bytes
from pngutil import chunk, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def switches(L):
    assert L.set_png_interlaced(1) == 0
    L.set_png_lossy(1); L.set_png_resize(1); L.set_webp_lossless_convert(1)
    yield
    L.set_png_interlaced(0); L.set_png_lossy(0); L.set_png_resize(0); L.set_webp_lossless_convert(0)


def _params(L, **kw):
    p = L.default_params()
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _legs(L, w, h, limit):
    """limit: compress_to_size's target, below both files' sizes (a source that fits is handed back as it is)"""
    tw = max(1, (w + 1) // 2)
    return [
        ("lossless_l0", lambda d: L.compress_in_memory(d, _params(L, png_optimize=1, png_optimization_level=0))),
        ("lossless_l3", lambda d: L.compress_in_memory(d, _params(L, png_optimize=1, png_optimization_level=3))),
        ("lossless_l6", lambda d: L.compress_in_memory(d, _params(L, png_optimize=1, png_optimization_level=6))),
        ("lossy_q80", lambda d: L.compress_in_memory(d, _params(L, png_optimize=0, png_quality=80))),
        ("resize", lambda d: L.compress_in_memory(d, _params(L, png_optimize=1, width=tw))),
        ("to_size", lambda d: L.compress_to_size_in_memory(d, _params(L, png_optimize=0), limit)),
        ("webp_lossless", lambda d: L.convert_in_memory(d, _params(L, webp_lossless=1), L.FMT_WEBP)),
        ("webp_lossy", lambda d: L.convert_in_memory(d, _params(L), L.FMT_WEBP)),
        ("jpeg", lambda d: L.convert_in_memory(d, _params(L), L.FMT_JPEG)),
        ("resize_samples", lambda d: (lambda r: (r[0].width, r[0].height, r[0].color_type, r[0].bit_depth, r[1].tobytes()))(L.png_resize_samples(d, tw, 0))),
    ]


def _run(call, data):
    try:
        return call(data)
    except Exception as e:                  # a refusal must be the twin's refusal, code and message
        return ("error", getattr(e, "code", None), str(e))


def _rgba(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data)); im.load()
    return np.asarray(im.convert("RGBA"))


def _check_twin(L, inter, twin, w, h, bd):
    for name, call in _legs(L, w, h, min(len(inter), len(twin)) - 1):
        a, b = _run(call, inter), _run(call, twin)
        assert a == b, name
        if name.startswith("lossless") and bd <= 8 and isinstance(a, bytes):
            assert np.array_equal(_rgba(a), _rgba(inter)), name


@pytest.mark.parametrize("ct,bd", pairs(), ids=lambda v: str(v))
@pytest.mark.parametrize("trns", [False, True], ids=["plain", "trns"])
def test_twin_property_every_pair(L, ct, bd, trns):
    if trns and ct in (4, 6):
        pytest.skip("colour types with an alpha channel carry no tRNS")
    form = ("key" if ct in (0, 2) else "partial") if trns else None
    for w, h in SHAPES + [(1023, 769)]:
        inter, twin, _, _, _ = adam7_case(w, h, ct, bd, seed=w * 13 + h + ct * 7 + bd, trns=form)
        _check_twin(L, inter, twin, w, h, bd)


def test_twin_property_photographs(L):
    for ct, bd in ((2, 8), (6, 8), (0, 8), (3, 8), (4, 8)):
        nc = CHANNELS[ct]
        img = synth(301, 257, nc, seed=ct, kind="photo" if ct != 3 else "flat")
        plte = b""
        if ct == 3:
            img = (img[..., 0] // 16).astype(np.uint8)[..., None]
            plte = bytes(np.random.default_rng(1).integers(0, 256, 48, dtype=np.uint8))
        inter, twin = adam7_pair(img.reshape(301, -1), 257, 301, ct, bd, seed=ct, plte=plte)
        _check_twin(L, inter, twin, 257, 301, bd)


def test_twin_property_4k_rgba(L):
    img = synth(4096, 4096, 4, seed=7)
    inter, twin = adam7_pair(img.reshape(4096, -1), 4096, 4096, 6, 8, seed=7, level=1)
    _check_twin(L, inter, twin, 4096, 4096, 8)


def test_batch_mixes_adam7_plain_and_jpeg(L, golden):
    items = []
    for k, (ct, bd) in enumerate(((2, 8), (0, 1), (6, 16), (3, 4))):
        inter, twin, _, _, _ = adam7_case(57 + k, 33 + 2 * k, ct, bd, seed=k, trns="partial" if ct == 3 else None)
        items += [inter, twin]
    jpg = golden("in_420_base_355x237.jpg")
    items.insert(3, jpg)
    for p in (_params(L, png_optimize=1), _params(L, png_optimize=0)):
        res = L.compress_batch(items, p, n_threads=4)
        assert all(r[1] == 0 for r in res), [r[1:] for r in res]
        outs = [r[0] for r in res]
        assert outs[3] == L.compress_in_memory(jpg, p)
        pngs = outs[:3] + outs[4:]
        for i in range(0, len(pngs), 2):
            assert pngs[i] == pngs[i + 1] == L.compress_in_memory(items[i + (i >= 3)], p)


# ---- damaged Adam7 files answer as their non-interlaced twins do ----------------------------------------------------------------

W, H, CT, BD = 37, 29, 2, 8


def _frame(z, interlace):
    ihdr = chunk(b"IHDR", W.to_bytes(4, "big") + H.to_bytes(4, "big") + bytes([BD, CT, 0, 0, interlace]))
    return b"\x89PNG\r\n\x1a\n" + ihdr + chunk(b"IDAT", z) + chunk(b"IEND", b"")


def _damaged():
    """(Adam7 file, non-interlaced file) with the same fault"""
    raw = np.random.default_rng(9).integers(0, 256, (H, row_bytes(W, CT, BD)), dtype=np.uint8)
    inter = bytearray(adam7_filtered(raw, W, H, CT, BD, seed=9))
    plain = bytearray(np.concatenate([np.zeros((H, 1), np.uint8), raw], 1).tobytes())
    passes, _, _ = layout(W, H, CHANNELS[CT] * BD)
    bad_i = bytearray(inter); bad_i[passes[4][3]] = 7                         # a pass-5 row's filter byte
    bad_p = bytearray(plain); bad_p[5 * (row_bytes(W, CT, BD) + 1)] = 7
    zi, zp = zlib.compress(bytes(inter)), zlib.compress(bytes(plain))
    flip = lambda z: z[:-4] + bytes([z[-4] ^ 1]) + z[-3:]
    cut = passes[5][3] + 10                                                   # ends inside pass 6
    return {
        "filter_byte": (_frame(zlib.compress(bytes(bad_i)), 1), _frame(zlib.compress(bytes(bad_p)), 0)),
        "adler": (_frame(flip(zi), 1), _frame(flip(zp), 0)),
        "truncated_in_pass_6": (_frame(zlib.compress(bytes(inter[:cut])), 1), _frame(zlib.compress(bytes(plain[:cut])), 0)),
    }


@pytest.mark.parametrize("fault", ["filter_byte", "adler", "truncated_in_pass_6"])
def test_damage_answers_like_the_twin(L, fault):
    inter, plain = _damaged()[fault]
    for name, call in _legs(L, W, H, 64) + [("decode", L.png_decode)]:
        a, b = _run(call, inter), _run(call, plain)
        assert a[0] == b[0] == "error" and a[1] == b[1] == 4, (name, a[:2], b[:2])
