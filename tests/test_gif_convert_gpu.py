"""Conversions to and from GIF on the device (b200_set_gif_convert), byte for byte: a GIF target equals the GIF leg's twin on the
canvas of the source's pixels; a GIF source's frame 0 takes the JPEG, PNG and WebP back ends exactly as the oracle does."""
import concurrent.futures
import io
import os
import subprocess
import zlib

import numpy as np
import pytest

import gif_cases
import gifutil
from gif_convert_cases import canvas, first_frame, twin
from oracle import gif as G
from png_webp_cases import cases as png_cases, expected_rgba, make_case
from pngutil import frame_png, pil_pixels, pil_png, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FMT_JPEG, FMT_PNG, FMT_GIF, FMT_WEBP = 0, 1, 2, 3
JPEGS = ["in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_gray_base_355x237.jpg", "in_420_prog_355x237.jpg"]


@pytest.fixture(autouse=True)
def switch_on(L):
    assert L.set_gif_convert(1) == 0
    yield
    L.set_gif_convert(0)


def _params(L, q=80, w=0, h=0):
    p = L.default_params(); p.gif_quality = q; p.width, p.height = w, h
    return p


def _opaque(rgb):
    return np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], axis=2)


def _jpeg_rgba(O, data):
    """the oracle's RGB decode of the lossy conversions (a grey source repeated), opaque"""
    ycc = O.Jpeg(data).decode_native()
    rgb = O.ycc_to_rgb(ycc) if ycc.shape[0] == 3 else np.repeat(ycc, 3, axis=0)
    return _opaque(np.ascontiguousarray(rgb.transpose(1, 2, 0)))


def _pil_rgba(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data)); im.load()
    return np.asarray(im.convert("RGBA"))


# ---- to GIF ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("q", [1, 50, 80, 100])
@pytest.mark.parametrize("name", JPEGS)
def test_jpeg_to_gif_equals_twin(L, O, golden, name, q):
    data = golden(name)
    assert L.convert_in_memory(data, _params(L, q), FMT_GIF) == twin(_jpeg_rgba(O, data), q)


@pytest.mark.parametrize("case", png_cases(), ids=lambda c: c[0])
def test_png_to_gif_equals_twin(L, case):
    _, w, h, ct, bd, trns, plte_len = case
    data, raw, plte, t = make_case(w, h, ct, bd, seed=w * 31 + h * 7 + ct * 5 + bd, trns=trns, plte_len=plte_len)
    want = expected_rgba(raw, w, ct, bd, plte, t)
    for q in (80, 100):
        assert L.convert_in_memory(data, _params(L, q), FMT_GIF) == twin(want, q), q


def test_png_partial_alpha_to_gif(L):
    img = synth(37, 53, 4, seed=4)
    img[..., 3] = np.array([0, 1, 254, 255])[np.add.outer(np.arange(37), np.arange(53)) % 4]
    data = pil_png(img)
    for q in (1, 60, 100):
        out = L.convert_in_memory(data, _params(L, q), FMT_GIF)
        assert out == twin(img, q), q
    shown = gifutil.decode(out)[0][0][0]
    assert np.array_equal(shown[..., 3] == 0, img[..., 3] == 0)


def test_webp_to_gif_equals_twin(L):
    from PIL import Image
    h, w = 70, 90
    rgba = synth(h, w, 4, seed=5)
    a = rgba[..., 3]
    rgba[..., 3] = np.where(a < 80, 0, np.where(a > 170, 255, a))          # clear, translucent and opaque pixels
    files = {}
    b = io.BytesIO(); Image.fromarray(rgba[..., :3].copy()).save(b, "WEBP", quality=80); files["lossy"] = b.getvalue()
    b = io.BytesIO(); Image.fromarray(rgba[..., :3].copy()).save(b, "WEBP", lossless=True); files["lossless"] = b.getvalue()
    b = io.BytesIO(); Image.fromarray(rgba).save(b, "WEBP", quality=80, alpha_quality=100); files["lossy_alpha"] = b.getvalue()
    b = io.BytesIO(); Image.fromarray(rgba).save(b, "WEBP", lossless=True, exact=True); files["lossless_alpha"] = b.getvalue()
    with open(os.path.join(ROOT, "tests", "golden", "reference_samples", "w0.webp"), "rb") as f:
        files["w0"] = f.read()
    for name, data in files.items():
        want = _pil_rgba(data)
        if name.endswith("alpha"):
            assert (want[..., 3] == 0).any() and (want[..., 3] == 255).any()
        for q in (50, 100):
            assert L.convert_in_memory(data, _params(L, q), FMT_GIF) == twin(want, q), (name, q)


def test_palette_png_equals_gif_reencode(L):
    """a PNG of at most 256 colours converts to the file the GIF leg writes for a one-frame GIF of the same pixels"""
    rng = np.random.default_rng(9)
    h, w = 61, 47
    idx = (np.add.outer(np.arange(h) // 5, np.arange(w) // 3) % 200).astype(np.uint8)
    table = [tuple(int(v) for v in c) for c in rng.integers(0, 256, (200, 3))]
    png = pil_png(gif_cases._pal_image(idx, table), transparency=bytes([0] + [255] * 199))
    gif = gif_cases.raw_gif(w, h, [dict(x=0, y=0, idx=idx, table=table, transparent=0)])
    try:
        assert L.set_gif(1) == 0
        for q in (30, 80, 100):
            assert L.convert_in_memory(png, _params(L, q), FMT_GIF) == L.compress_in_memory(gif, _params(L, q)), q
    finally:
        L.set_gif(0)


def test_large_png_equals_twin(L):
    img = synth(1500, 2000, 3, seed=12)
    assert L.convert_in_memory(pil_png(img), _params(L, 70), FMT_GIF) == twin(_opaque(img), 70)


def test_24mp_jpeg_to_gif(L, O):
    from PIL import Image
    b = io.BytesIO(); Image.fromarray(synth(1000, 1500, 3, seed=13)).resize((6000, 4000)).save(b, "JPEG", quality=90); data = b.getvalue()
    out = L.convert_in_memory(data, _params(L, 80), FMT_GIF)
    assert out[:6] == b"GIF89a" and int.from_bytes(out[6:8], "little") == 6000 and int.from_bytes(out[8:10], "little") == 4000
    pal, idx = G.gif_quantize(canvas(_jpeg_rgba(O, data)), 80)
    assert np.array_equal(_pil_rgba(out)[..., :3], pal[idx][..., :3])


# ---- from GIF --------------------------------------------------------------------------------------------------------------------
GIFS = [(n, d) for n, d in gif_cases.cases() if n in ("still_m2", "still_m8", "still_interlaced", "anim_disposal2", "anim_opaque", "disposal_mix", "g1")]


def _planar(rgba):
    return np.ascontiguousarray(rgba[..., :3].transpose(2, 0, 1))


@pytest.mark.parametrize("tw,th", [(0, 0), (40, 0), (0, 250)])
@pytest.mark.parametrize("name,data", GIFS, ids=[n for n, _ in GIFS])
def test_gif_to_jpeg(L, O, name, data, tw, th):
    f0 = first_frame(data)
    h, w = f0.shape[:2]
    p = L.default_params(); p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = 85, 420, 1
    p.width, p.height = tw, th
    op = O.params(85, 420, True)
    rgb = _planar(f0)
    if tw or th:
        nw, nh = O.compute_dimensions(w, h, tw, th)
        rgb = np.stack([O.resize_plane(np.ascontiguousarray(rgb[c]), nw, nh) for c in range(3)])
    assert L.convert_in_memory(data, p, FMT_JPEG) == O.write(O.forward(O.rgb_to_ycc(rgb), op), op)


@pytest.mark.parametrize("name,data", GIFS, ids=[n for n, _ in GIFS])
def test_gif_to_png(L, O, name, data):
    f0 = first_frame(data)
    h, w = f0.shape[:2]
    clear = (f0[..., 3] == 0).any()
    mode = "RGBA" if clear else "RGB"
    p = L.default_params(); p.png_optimize = 1
    got = pil_pixels(L.convert_in_memory(data, p, FMT_PNG))
    assert ("A" in got.mode or "transparency" in got.info) == clear
    assert np.array_equal(np.asarray(got.convert(mode)), f0[..., :len(mode)])
    p.width = 29
    nw, nh = O.compute_dimensions(w, h, 29, 0)
    got = np.asarray(pil_pixels(L.convert_in_memory(data, p, FMT_PNG)).convert(mode))
    want = np.stack([O.resize_plane(np.ascontiguousarray(f0[..., c]), nw, nh) for c in range(len(mode))], axis=-1)
    assert np.array_equal(got, want)


def _chunks(f):
    out, pos = {}, 12
    while pos < len(f):
        n = int.from_bytes(f[pos + 4:pos + 8], "little")
        out[f[pos:pos + 4]] = f[pos + 8:pos + 8 + n]
        pos += 8 + n + (n & 1)
    return out


@pytest.mark.parametrize("name,data", GIFS, ids=[n for n, _ in GIFS])
def test_gif_to_webp(L, O, name, data):
    f0 = first_frame(data)
    h, w = f0.shape[:2]
    p = L.default_params(); p.webp_quality = 75
    out = L.convert_in_memory(data, p, FMT_WEBP)
    frame = O.webp_encode(_planar(f0), 75)[0]
    a = np.ascontiguousarray(f0[..., 3])
    if not (a == 0).any():
        assert out == frame
        return
    ch = _chunks(out)
    assert set(ch) == {b"VP8X", b"ALPH", b"VP8 "} and ch[b"VP8 "] == _chunks(frame)[b"VP8 "]
    k, res = L.webp_alpha_filter(a)
    tok, _ = O.png_lz77(res.reshape(-1), 1, w)
    assert ch[b"ALPH"] == L.webp_alpha_chunk(tok, w, h, k)
    assert np.array_equal(_pil_rgba(out)[..., 3], a)


# ---- refusals, threads, CLI ------------------------------------------------------------------------------------------------------
def _code(L, data, p, fmt):
    with pytest.raises(L.B200Error) as e:
        L.convert_in_memory(data, p, fmt)
    return e.value.code, str(e.value)


def test_refusals(L, golden):
    jpg, png, gif = golden("in_420_base_355x237.jpg"), pil_png(synth(20, 30, 3, seed=1)), dict(gif_cases.cases())["anim_disposal1"]
    b = io.BytesIO()
    from PIL import Image
    Image.fromarray(synth(20, 30, 3, seed=2)).save(b, "WEBP"); webp = b.getvalue()
    pj = L.default_params(); pp = L.default_params(); pp.png_optimize = 1
    routes = [(jpg, FMT_GIF, pj), (png, FMT_GIF, pj), (webp, FMT_GIF, pj), (gif, FMT_JPEG, pj), (gif, FMT_PNG, pp), (gif, FMT_WEBP, pj)]
    L.set_gif_convert(0)
    for data, fmt, p in routes:
        assert _code(L, data, p, fmt)[0] == 3
    L.set_gif_convert(1)
    for data, fmt, p in routes:
        L.convert_in_memory(data, p, fmt)
    for data in (jpg, png, webp):
        assert _code(L, data, _params(L, 80, 10, 0), FMT_GIF) == (3, "GIF resize is outside the GPU path (route to caesium::convert_in_memory) [3]")
    lossless = L.default_params(); lossless.webp_lossless = 1
    assert _code(L, gif, lossless, FMT_WEBP)[0] == 3
    assert _code(L, gif, L.default_params(), FMT_PNG)[0] == 3              # lossy PNG while its switch is off
    assert _code(L, gif[:100], pj, FMT_JPEG)[0] == 4
    assert _code(L, jpg[:200], pj, FMT_GIF)[0] == 4
    bad_png = bytearray(png); bad_png[-20] ^= 0xFF
    assert _code(L, bytes(bad_png), pj, FMT_GIF)[0] == 4
    _, raw, _, _ = make_case(20, 9, 2, 8, seed=4)
    filt = np.concatenate([np.zeros((9, 1), np.uint8), raw], axis=1)
    filt[5, 0] = 7                                                          # a filter byte the device un-filter refuses
    assert _code(L, frame_png(20, 9, 8, 2, zlib.compress(filt.tobytes())), pj, FMT_GIF)[0] == 4
    assert _code(L, webp[:len(webp) // 2], pj, FMT_GIF)[0] == 4
    assert _code(L, gif, pj, FMT_GIF)[0] == 8
    assert _code(L, b"garbage", pj, FMT_GIF)[0] == 2
    past = gif_cases.raw_gif(6, 2, [dict(x=3, y=0, idx=np.zeros((2, 4), np.uint8), table=[(0, 0, 0), (1, 1, 1)], m=2)])
    assert _code(L, past, pj, FMT_JPEG)[0] == 3


def _mixed(golden):
    from PIL import Image
    b = io.BytesIO(); Image.fromarray(synth(70, 90, 4, seed=3)).save(b, "WEBP", lossless=True); webp = b.getvalue()
    g = dict(gif_cases.cases())
    return [(golden("in_420_base_640x480.jpg"), FMT_GIF), (pil_png(synth(123, 77, 4, seed=4)), FMT_GIF), (webp, FMT_GIF),
            (golden("in_gray_base_355x237.jpg"), FMT_GIF), (g["g1"], FMT_WEBP), (g["disposal_mix"], FMT_JPEG), (g["anim_disposal3"], FMT_WEBP),
            (make_case(301, 157, 3, 4, seed=5, trns="partial")[0], FMT_GIF)]


def test_threads_equal_serial(L, golden):
    items = _mixed(golden) * 3
    p = _params(L, 70)
    serial = [L.convert_in_memory(d, p, f) for d, f in items]
    with concurrent.futures.ThreadPoolExecutor(8) as ex:
        par = list(ex.map(lambda it: L.convert_in_memory(it[0], p, it[1]), items))
    assert par == serial


def test_cli_writes_convert_in_memory_bytes(L, golden, tmp_path):
    exe = os.path.join(ROOT, "caesium-clt_b200", "b200clt")
    src = tmp_path / "in"; src.mkdir()
    jpg, gif = golden("in_420_base_640x480.jpg"), dict(gif_cases.cases())["g1"]
    (src / "a.jpg").write_bytes(jpg); (src / "b.gif").write_bytes(gif)
    env = dict(os.environ, B200_GIF_CONVERT="gpu")
    out = tmp_path / "gif"
    r = subprocess.run([exe, "-q", "80", "--format", "gif", "-o", str(out), str(src / "a.jpg")], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    assert (out / "a.gif").read_bytes() == L.convert_in_memory(jpg, L.default_params(), FMT_GIF)
    out = tmp_path / "webp"
    r = subprocess.run([exe, "-q", "80", "--format", "webp", "-o", str(out), str(src / "b.gif")], capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    assert (out / "b.webp").read_bytes() == L.convert_in_memory(gif, L.default_params(), FMT_WEBP)
