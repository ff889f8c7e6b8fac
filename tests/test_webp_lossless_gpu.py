"""GPU parity tests of the lossless WebP (VP8L) leg: compress_in_memory with webp_lossless on WebP sources runs the device encoder
(vp8l_kernels.cu + vp8l_encode.cpp) and must write the oracle's file (oracle/vp8l_oracle.c) byte for byte; every output must decode
through libwebp (Pillow) to exactly the decoded source."""
import io
import json
import os
import subprocess

import numpy as np
import pytest

from pngutil import pil_png, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def OV(O):
    """the lossless WebP encoder twin (oracle/vp8l.py over oracle/vp8l_oracle.c)"""
    from oracle import vp8l
    return vp8l


def _sample(name):
    with open(os.path.join(ROOT, "tests", "golden", "reference_samples", name), "rb") as f:
        return f.read()


def _soft_alpha(h, w, seed):
    yy, xx = np.mgrid[:h, :w]
    a = np.clip(300 - np.hypot(yy - h / 2, xx - w / 2) * 600 / max(h, w), 0, 255).astype(np.uint8)
    a[: h // 8] = 0
    rng = np.random.default_rng(seed)
    a[h // 2:h // 2 + 4] = rng.integers(0, 256, (min(4, h - h // 2), w), dtype=np.uint8)
    return a


def _webp(img, **kw):
    from PIL import Image
    b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", **kw)
    return b.getvalue()


def _decoded_rgba(L, data):
    rgb, a = L.webp_decode_rgba(data)
    if a is None:
        a = np.full(rgb.shape[:2], 255, np.uint8)
    return np.ascontiguousarray(np.concatenate([rgb, a[:, :, None]], axis=2))


def _pil_rgba(data):
    from PIL import Image
    im = Image.open(io.BytesIO(data))
    assert im.format == "WEBP"
    return np.asarray(im.convert("RGBA"))


def _params(L, **kw):
    p = L.default_params(); p.webp_lossless = 1
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _sources():
    h, w = 150, 210
    photo = synth(h, w, 3, seed=12, kind="photo")
    rgba = np.concatenate([photo, _soft_alpha(h, w, 3)[:, :, None]], axis=2)
    rgba[:20, :, :3] = 77                                   # colour under alpha 0 (rows 0..17 are fully transparent)
    yield "vp8", _webp(photo, quality=80)
    yield "vp8_odd", _webp(synth(37, 53, 3, seed=4, kind="flat"), quality=60)
    yield "vp8l_rgb", _webp(synth(97, 131, 3, seed=5, kind="flat"), lossless=True)
    yield "vp8l_rgba_exact", _webp(rgba, lossless=True, exact=True)
    yield "vp8x_alph", _webp(rgba, quality=85, alpha_quality=100)
    yield "w0", _sample("w0.webp")
    yield "w1", _sample("w1.webp")


@pytest.mark.parametrize("case", list(_sources()), ids=lambda c: c[0])
def test_lossless_webp_matches_oracle_and_round_trips(L, OV, case):
    _, src = case
    want_px = _decoded_rgba(L, src)
    out = L.compress_in_memory(src, _params(L))
    assert out == OV.webp_lossless_encode(want_px)
    assert out[12:16] == b"VP8L" and int.from_bytes(out[4:8], "little") == len(out) - 8
    assert np.array_equal(_pil_rgba(out), want_px)
    assert bool(out[20 + 4] & 0x10) == bool((want_px[:, :, 3] != 255).any())     # alpha_is_used iff some alpha is not 255


@pytest.mark.parametrize("kind", ["photo", "flat"])
def test_lossless_webp_4k(L, OV, kind):
    img = synth(2160, 3840, 3, seed=7, kind=kind)
    src = _webp(img, lossless=True, method=0)
    px = _decoded_rgba(L, src)
    out = L.compress_in_memory(src, _params(L))
    assert out == OV.webp_lossless_encode(px)
    assert np.array_equal(_pil_rgba(out), px)


def test_lossless_webp_resize(L, O, OV):
    h, w = 150, 210
    rgba = np.concatenate([synth(h, w, 3, seed=2, kind="photo"), _soft_alpha(h, w, 1)[:, :, None]], axis=2)
    for src in (_webp(rgba, lossless=True, exact=True), _webp(rgba[:, :, :3].copy(), quality=90)):
        px = _decoded_rgba(L, src)
        opaque = bool((px[:, :, 3] == 255).all())
        nw, nh = O.compute_dimensions(w, h, 100, 0)
        out = L.compress_in_memory(src, _params(L, width=100))
        planes = [O.resize_plane(np.ascontiguousarray(px[:, :, c]), nw, nh) for c in range(3)]
        planes.append(np.full((nh, nw), 255, np.uint8) if opaque else O.resize_plane(np.ascontiguousarray(px[:, :, 3]), nw, nh))
        want = np.ascontiguousarray(np.stack(planes, -1))
        assert out == OV.webp_lossless_encode(want)
        assert np.array_equal(_pil_rgba(out), want)


def test_lossless_webp_repeated_calls_of_different_sizes(L, OV):
    srcs = [_webp(synth(h, w, 3, seed=h, kind=k), lossless=True) for h, w, k in ((400, 600, "photo"), (1, 1, "flat"), (33, 17, "photo"), (400, 600, "flat"), (5, 900, "photo"))]
    want = [OV.webp_lossless_encode(_decoded_rgba(L, s)) for s in srcs]
    for _ in range(2):
        for s, wnt in zip(srcs, want):
            assert L.compress_in_memory(s, _params(L)) == wnt


def test_lossless_batch_mixed_formats(L, golden):
    srcs = [golden("in_420_base_640x480.jpg"), pil_png(synth(64, 96, 3, seed=1)), _webp(synth(80, 120, 3, seed=3), quality=80),
            _webp(synth(45, 70, 3, seed=8, kind="flat"), lossless=True), golden("in_420_tiny_17x9.jpg"), _sample("w0.webp")]
    p = L.default_params(); p.jpeg_optimize = p.png_optimize = p.webp_lossless = 1
    res = L.compress_batch(srcs, p)
    for s, (data, code, msg) in zip(srcs, res):
        assert code == 0, msg
        assert data == L.compress_in_memory(s, p)


def test_cli_lossless_on_webp_files(L, tmp_path):
    exe = os.path.join(ROOT, "caesium-clt_b200", "b200clt")
    src = tmp_path / "in"; src.mkdir()
    (src / "a.webp").write_bytes(_webp(synth(64, 96, 3, seed=1), quality=80))
    (src / "b.webp").write_bytes(_sample("w1.webp"))
    (src / "c.png").write_bytes(pil_png(synth(40, 50, 3, seed=2)))
    out = tmp_path / "out"
    r = subprocess.run([exe, "--lossless", "--json", "-o", str(out), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    files = json.loads(r.stdout)["files"]
    assert {os.path.basename(f["original_path"]) for f in files if f["status"] == "success"} >= {"a.webp", "b.webp", "c.png"}
    p = _params(L)
    for name in ("a.webp", "b.webp"):
        assert (out / name).read_bytes() == L.compress_in_memory((src / name).read_bytes(), p)
