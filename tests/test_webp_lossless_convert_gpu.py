"""JPEG / PNG -> lossless WebP on the device (b200_set_webp_lossless_convert): every file equals the oracle's VP8L encoding of the pixels
the lossy conversion feeds its encoder, and libwebp decodes it back to exactly those pixels."""
import concurrent.futures
import io
import os
import subprocess
import zlib

import numpy as np
import pytest

from png_webp_cases import cases, expected_rgba, make_case
from pngutil import chunk, frame_png, pil_png, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JPEGS = ["in_420_base_355x237.jpg", "in_420_prog_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg",
         "in_gray_base_355x237.jpg", "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"]


@pytest.fixture(scope="module", autouse=True)
def switch_on(L):
    assert L.set_webp_lossless_convert(1) == 0
    yield
    L.set_webp_lossless_convert(0)


@pytest.fixture(scope="module")
def OV(O):
    from oracle import vp8l
    return vp8l


def _params(L, w=0, h=0, lossless=1):
    p = L.default_params(); p.webp_lossless = lossless; p.width, p.height = w, h
    return p


def _pil_rgba(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data)); im.load()
    return np.asarray(im.convert("RGBA"))


def _jpeg_rgba(O, data, nw=None, nh=None):
    """_jpeg_rgb of the lossy conversion's tests (oracle decode, YCbCr -> RGB, Lanczos3 per plane) with alpha 255"""
    ycc = O.Jpeg(data).decode_native()
    rgb = O.ycc_to_rgb(ycc) if ycc.shape[0] == 3 else np.repeat(ycc, 3, axis=0)
    if nw is not None and (nw, nh) != (rgb.shape[2], rgb.shape[1]):
        rgb = np.stack([O.resize_plane(rgb[c], nw, nh) for c in range(3)])
    rgba = np.concatenate([rgb.transpose(1, 2, 0), np.full(rgb.shape[1:] + (1,), 255, np.uint8)], axis=2)
    return np.ascontiguousarray(rgba)


def _png_rgba(L, O, data, plte, trns, nw=None, nh=None):
    """the restatement over the host decoder's rows; resized per 8-bit plane, alpha only when translucent"""
    info, raw = L.png_decode(data)
    rgba = expected_rgba(raw, info.width, info.color_type, info.bit_depth, plte, trns)
    if nw is not None and (nw, nh) != (info.width, info.height):
        translucent = (rgba[..., 3] != 255).any()
        planes = [O.resize_plane(np.ascontiguousarray(rgba[..., c]), nw, nh) for c in range(4 if translucent else 3)]
        if not translucent:
            planes.append(np.full((nh, nw), 255, np.uint8))
        rgba = np.stack(planes, axis=-1)
    return np.ascontiguousarray(rgba)


def _check(out, OV, rgba):
    assert out == OV.webp_lossless_encode(rgba)
    assert np.array_equal(_pil_rgba(out), rgba)


@pytest.mark.parametrize("name", JPEGS)
def test_jpeg_matches_oracle(L, O, OV, golden, name):
    data = golden(name)
    _check(L.convert_in_memory(data, _params(L), L.FMT_WEBP), OV, _jpeg_rgba(O, data))


@pytest.mark.parametrize("tw,th", [(200, 0), (0, 100), (177, 99), (900, 0)])
def test_jpeg_resized_matches_oracle(L, O, OV, golden, tw, th):
    data = golden("in_420_base_640x480.jpg")
    nw, nh = O.compute_dimensions(640, 480, tw, th)
    _check(L.convert_in_memory(data, _params(L, tw, th), L.FMT_WEBP), OV, _jpeg_rgba(O, data, nw, nh))


@pytest.mark.parametrize("case", cases(), ids=lambda c: c[0])
def test_png_matches_oracle(L, O, OV, case):
    _, w, h, ct, bd, trns, plte_len = case
    data, raw, plte, t = make_case(w, h, ct, bd, seed=w * 31 + h * 7 + ct * 5 + bd, trns=trns, plte_len=plte_len)
    assert np.array_equal(L.png_decode(data)[1], raw)
    _check(L.convert_in_memory(data, _params(L), L.FMT_WEBP), OV, _png_rgba(L, O, data, plte, t))


RESIZE_CASES = [c for c in cases() if c[1] == 13]


@pytest.mark.parametrize("case", RESIZE_CASES, ids=lambda c: c[0])
def test_png_resized_matches_oracle(L, O, OV, case):
    _, w, h, ct, bd, trns, plte_len = case
    data, raw, plte, t = make_case(w, h, ct, bd, seed=w * 31 + h * 7 + ct * 5 + bd, trns=trns, plte_len=plte_len)
    for tw, th in ((8, 0), (0, 15), (29, 3)):
        nw, nh = O.compute_dimensions(w, h, tw, th)
        _check(L.convert_in_memory(data, _params(L, tw, th), L.FMT_WEBP), OV, _png_rgba(L, O, data, plte, t, nw, nh))


def _soft_rgba(h, w, seed):
    img = synth(h, w, 4, seed=seed, kind="photo")
    yy, xx = np.mgrid[:h, :w]
    img[..., 3] = np.clip(300 - np.hypot(yy - h / 2, xx - w / 2) * 600 / w, 0, 255).astype(np.uint8)
    img[: h // 4, : w // 4, 3] = 0                                  # colour under alpha 0 is kept
    return img


@pytest.mark.parametrize("kind", ["rgba_soft", "rgba_opaque", "rgb_pillow", "la_pillow", "palette_pillow"])
def test_pillow_pngs(L, O, OV, kind):
    from PIL import Image
    h, w = 61, 83
    if kind == "rgba_soft":
        data = pil_png(_soft_rgba(h, w, 5))
    elif kind == "rgba_opaque":
        img = synth(h, w, 4, seed=6); img[..., 3] = 255; data = pil_png(img)
    elif kind == "rgb_pillow":
        data = pil_png(synth(h, w, 3, seed=7, kind="flat"))
    elif kind == "la_pillow":
        data = pil_png(synth(h, w, 2, seed=8))
    else:
        data = pil_png(Image.fromarray(synth(h, w, 3, seed=9, kind="flat")).quantize(17))
    want = _pil_rgba(data)                                          # 8-bit sources: Pillow's own decode is the rule
    out = L.convert_in_memory(data, _params(L), L.FMT_WEBP)
    _check(out, OV, want)
    if kind == "rgba_opaque":
        assert out[20:21] == b"\x2f" and (out[21 + 3] >> 4) & 1 == 0          # VP8L header: alpha_is_used = 0
    for tw, th in ((40, 0), (0, 100)):
        nw, nh = O.compute_dimensions(w, h, tw, th)
        translucent = (want[..., 3] != 255).any()
        planes = [O.resize_plane(np.ascontiguousarray(want[..., c]), nw, nh) for c in range(4 if translucent else 3)]
        if not translucent:
            planes.append(np.full((nh, nw), 255, np.uint8))
        _check(L.convert_in_memory(data, _params(L, tw, th), L.FMT_WEBP), OV, np.ascontiguousarray(np.stack(planes, -1)))


def test_4k_parity(L, O, OV):
    from PIL import Image
    img = synth(2160, 3840, 3, seed=11)
    b = io.BytesIO(); Image.fromarray(img).save(b, "JPEG", quality=90); jpg = b.getvalue()
    _check(L.convert_in_memory(jpg, _params(L), L.FMT_WEBP), OV, _jpeg_rgba(O, jpg))
    png = pil_png(img)
    _check(L.convert_in_memory(png, _params(L), L.FMT_WEBP), OV, np.ascontiguousarray(np.concatenate([img, np.full(img.shape[:2] + (1,), 255, np.uint8)], 2)))


def test_dimension_limit(L, O, OV):
    row = np.random.default_rng(3).integers(0, 256, (1, 16383), dtype=np.uint8)
    data = pil_png(row)
    _check(L.convert_in_memory(data, _params(L), L.FMT_WEBP), OV, np.ascontiguousarray(np.stack([row, row, row, np.full_like(row, 255)], -1)))
    wide = pil_png(np.zeros((1, 16384), np.uint8))
    with pytest.raises(L.B200Error) as lossless:
        L.convert_in_memory(wide, _params(L), L.FMT_WEBP)
    with pytest.raises(L.B200Error) as lossy:
        L.convert_in_memory(wide, _params(L, lossless=0), L.FMT_WEBP)
    assert lossless.value.code == lossy.value.code == 1 and str(lossless.value) == str(lossy.value)


def _broken():
    data, raw, _, _ = make_case(20, 9, 2, 8, seed=4)
    filt = np.concatenate([np.zeros((9, 1), np.uint8), raw], axis=1)
    bad_filter = filt.copy(); bad_filter[5, 0] = 7
    z = zlib.compress(filt.tobytes())
    return {
        "truncated_idat": frame_png(20, 9, 8, 2, zlib.compress(filt.tobytes()[:-40])),
        "bad_filter_byte": frame_png(20, 9, 8, 2, zlib.compress(bad_filter.tobytes())),
        "adler_mismatch": frame_png(20, 9, 8, 2, z[:-4] + bytes([z[-4] ^ 1]) + z[-3:]),
    }


def test_interlaced_and_corrupt_pngs(L):
    ihdr = chunk(b"IHDR", (5).to_bytes(4, "big") + (4).to_bytes(4, "big") + bytes([8, 0, 0, 0, 1]))
    inter = b"\x89PNG\r\n\x1a\n" + ihdr + chunk(b"IDAT", zlib.compress(bytes(64))) + chunk(b"IEND", b"")
    with pytest.raises(L.B200Error) as e:
        L.convert_in_memory(inter, _params(L), L.FMT_WEBP)
    assert e.value.code == 3
    for name, data in _broken().items():
        codes = []
        for lossless in (1, 0):
            with pytest.raises(L.B200Error) as e:
                L.convert_in_memory(data, _params(L, lossless=lossless), L.FMT_WEBP)
            codes.append(e.value.code)
        assert codes == [4, 4], name


def test_compress_to_size_stays_refused(L):
    from PIL import Image
    b = io.BytesIO(); Image.fromarray(synth(40, 50, 3, seed=2)).save(b, "WEBP", lossless=True); src = b.getvalue()
    with pytest.raises(L.B200Error) as e:
        L.compress_to_size_in_memory(src, _params(L), len(src) // 2)
    assert e.value.code == 3


def _mixed(golden):
    from PIL import Image
    b = io.BytesIO(); Image.fromarray(synth(70, 90, 3, seed=3)).save(b, "WEBP", lossless=True); webp = b.getvalue()
    return [("jpeg", golden("in_420_base_640x480.jpg"), 0), ("png_soft", pil_png(_soft_rgba(123, 77, 4)), 0), ("jpeg_small", golden("in_420_tiny_17x9.jpg"), 0),
            ("png_pal", make_case(301, 157, 3, 4, seed=5, trns="partial")[0], 0), ("jpeg_rz", golden("in_444_base_355x237.jpg"), 120),
            ("png_rz", pil_png(synth(211, 97, 3, seed=6)), 50), ("webp_src", webp, 0), ("png_grey16", make_case(57, 33, 0, 16, seed=7, trns="key")[0], 0)]


def _call(L, name, data, width):
    p = _params(L, width, 0)
    if name == "webp_src":
        return L.compress_in_memory(data, p)
    return L.convert_in_memory(data, p, L.FMT_WEBP)


def test_repeated_calls_interleaved(L, golden):
    """buffers left by larger or smaller calls, WebP-source lossless calls and lossy conversions change no later result"""
    items = _mixed(golden)
    first = [_call(L, n, d, w) for n, d, w in items]
    lossy = L.convert_in_memory(golden("in_420_base_355x237.jpg"), _params(L, lossless=0), L.FMT_WEBP)
    for k in range(3):
        for (n, d, w), f in list(zip(items, first))[::(-1) ** k]:
            assert _call(L, n, d, w) == f, n
            assert L.convert_in_memory(golden("in_420_base_355x237.jpg"), _params(L, lossless=0), L.FMT_WEBP) == lossy


def test_threads_equal_serial(L, golden):
    items = _mixed(golden) * 4
    serial = [_call(L, n, d, w) for n, d, w in items]
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        par = list(ex.map(lambda it: _call(L, *it), items))
    assert par == serial


def test_cli_writes_convert_in_memory_bytes(L, golden, tmp_path):
    exe = os.path.join(ROOT, "caesium-clt_b200", "b200clt")
    src = tmp_path / "in"; src.mkdir()
    jpg, png = golden("in_420_base_640x480.jpg"), pil_png(_soft_rgba(64, 96, 1))
    (src / "a.jpg").write_bytes(jpg); (src / "b.png").write_bytes(png)
    out = tmp_path / "out"
    env = dict(os.environ, B200_WEBP_LOSSLESS_CONVERT="gpu")
    r = subprocess.run([exe, "--lossless", "--format", "webp", "-o", str(out), str(src)], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    assert (out / "a.webp").read_bytes() == L.convert_in_memory(jpg, _params(L), L.FMT_WEBP)
    assert (out / "b.webp").read_bytes() == L.convert_in_memory(png, _params(L), L.FMT_WEBP)
