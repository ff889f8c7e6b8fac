"""GPU parity tests of the WebP (lossy VP8) leg, SURVEY.md §8 row a10: K8 (RGB -> YUV, intra prediction, forward DCT/WHT,
quantisation, reconstruction wavefront) + the host boolean coder, through the C-ABI, against the oracle.
Bar: bit-exact stage output (levels, modes) and byte-identical files; and independently of the oracle, libwebp must decode
the product's files to the reconstruction the stage output implies."""
import numpy as np
import pytest

from pngutil import pil_png, synth
from webputil import pil_decode

pytestmark = pytest.mark.gpu

FMT_JPEG, FMT_PNG, FMT_GIF, FMT_WEBP = 0, 1, 2, 3


def planar(img):
    return np.ascontiguousarray(img.transpose(2, 0, 1))


@pytest.mark.parametrize("h,w", [(64, 64), (37, 53), (1, 1), (16, 16), (17, 16), (16, 17), (15, 300), (300, 15), (129, 65), (240, 320)])
@pytest.mark.parametrize("q,kind", [(75, "photo"), (30, "flat"), (95, "noise"), (0, "photo"), (100, "flat")])
def test_k8_stage_and_file_match_oracle(L, O, h, w, q, kind):
    img = planar(synth(h, w, 3, seed=h * 7 + w + q, kind=kind))
    data, levels, modes = L.webp_encode_rgb(img, q, want_stage=True)
    wl, wm = O.webp_analyze(img, q)
    assert np.array_equal(modes, wm), "prediction modes / skip flags"
    assert np.array_equal(levels, wl), "quantised levels"
    want, _ = O.webp_encode(img, q)
    assert data == want


def test_k8_many_rows_wavefront(L, O):
    # tall and wide frames: hundreds of macroblock rows in flight, every row waits on the one above
    for h, w in ((2000, 48), (48, 2000), (1080, 1920)):
        img = planar(synth(h, w, 3, seed=h, kind="photo"))
        data = L.webp_encode_rgb(img, 80)
        want, _ = O.webp_encode(img, 80)
        assert data == want
        dec = pil_decode(data)
        assert dec.shape == (h, w, 3)
        assert np.abs(dec.astype(int) - img.transpose(1, 2, 0).astype(int)).mean() < 4.0


def test_k8_repeatable(L):
    img = planar(synth(333, 517, 3, seed=9, kind="photo"))
    a = L.webp_encode_rgb(img, 60)
    for _ in range(5):
        assert L.webp_encode_rgb(img, 60) == a


def _jpeg_rgb(O, data, nw=None, nh=None):
    """Oracle restatement of the convert front end: decode -> RGB -> (Lanczos3) ; planar [3, h, w]."""
    ycc = O.Jpeg(data).decode_native()
    rgb = O.ycc_to_rgb(ycc) if ycc.shape[0] == 3 else np.repeat(ycc, 3, axis=0)
    if nw is not None and (nw, nh) != (rgb.shape[2], rgb.shape[1]):
        rgb = np.stack([O.resize_plane(rgb[c], nw, nh) for c in range(3)])
    return rgb


@pytest.mark.parametrize("name", ["in_420_base_355x237.jpg", "in_420_prog_355x237.jpg", "in_444_base_355x237.jpg", "in_422_base_355x237.jpg",
                                  "in_gray_base_355x237.jpg", "in_420_base_640x480.jpg", "in_420_tiny_17x9.jpg", "in_420_tiny_3x3.jpg"])
def test_convert_jpeg_to_webp_matches_oracle(L, O, golden, name):
    data = golden(name)
    p = L.default_params(); p.webp_quality = 85
    out = L.convert_in_memory(data, p, FMT_WEBP)
    want, _ = O.webp_encode(_jpeg_rgb(O, data), 85)
    assert out == want
    assert pil_decode(out).shape[:2] == _jpeg_rgb(O, data).shape[1:]


@pytest.mark.parametrize("tw,th", [(200, 0), (0, 100), (177, 99), (640, 480)])
def test_convert_jpeg_to_webp_with_resize_matches_oracle(L, O, golden, tw, th):
    data = golden("in_420_base_640x480.jpg")
    p = L.default_params(); p.webp_quality = 70; p.width, p.height = tw, th
    out = L.convert_in_memory(data, p, FMT_WEBP)
    nw, nh = O.compute_dimensions(640, 480, tw, th)
    want, _ = O.webp_encode(_jpeg_rgb(O, data, nw, nh), 70)
    assert out == want


def test_convert_png_to_webp_matches_oracle(L, O):
    from PIL import Image
    rng = np.random.default_rng(2)
    rgb = synth(90, 120, 3, seed=4)
    p = L.default_params(); p.webp_quality = 80
    assert L.convert_in_memory(pil_png(rgb), p, FMT_WEBP) == O.webp_encode(planar(rgb), 80)[0]
    opaque = np.concatenate([rgb, np.full((90, 120, 1), 255, np.uint8)], axis=2)        # fully opaque alpha carries nothing
    assert L.convert_in_memory(pil_png(opaque), p, FMT_WEBP) == O.webp_encode(planar(rgb), 80)[0]
    grey = synth(50, 70, 1, seed=6)
    assert L.convert_in_memory(pil_png(grey), p, FMT_WEBP) == O.webp_encode(planar(np.repeat(grey, 3, axis=2)), 80)[0]
    idx = rng.integers(0, 16, (40, 60)).astype(np.uint8)
    im = Image.fromarray(idx, mode="P"); im.putpalette([int(v) for v in rng.integers(0, 256, 48)])
    want = O.webp_encode(planar(np.asarray(im.convert("RGB"))), 80)[0]
    assert L.convert_in_memory(pil_png(im), p, FMT_WEBP) == want


def test_convert_png_to_webp_with_resize_matches_oracle(L, O):
    rgb = synth(120, 200, 3, seed=8)
    p = L.default_params(); p.webp_quality = 75; p.width = 77
    nw, nh = O.compute_dimensions(200, 120, 77, 0)
    want = O.webp_encode(np.stack([O.resize_plane(np.ascontiguousarray(rgb[:, :, c]), nw, nh) for c in range(3)]), 75)[0]
    assert L.convert_in_memory(pil_png(rgb), p, FMT_WEBP) == want


@pytest.mark.parametrize("q,ss,prog", [(80, 0, True), (90, 444, False), (60, 422, True)])
def test_convert_png_to_jpeg_matches_oracle(L, O, q, ss, prog):
    """PNG -> JPEG: RGB -> YCbCr (jccolor tables) -> box downsample -> FDCT/quantise -> Huffman, all against the oracle's
    forward path (itself bit-exact with libjpeg-turbo, tests/test_oracle_jpeg.py)."""
    rgb = synth(93, 141, 3, seed=q)
    p = L.default_params(); p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = q, ss, int(prog)
    op = O.params(q, ss, prog)
    want = O.write(O.forward(O.rgb_to_ycc(planar(rgb)), op), op)
    assert L.convert_in_memory(pil_png(rgb), p, FMT_JPEG) == want
    grey = synth(50, 70, 1, seed=q)                                   # grey PNG -> single-component JPEG
    want = O.write(O.forward(planar(grey), op), op)
    assert L.convert_in_memory(pil_png(grey), p, FMT_JPEG) == want
    p.width = 64                                                      # with Lanczos3 resize
    nw, nh = O.compute_dimensions(141, 93, 64, 0)
    rz = np.stack([O.resize_plane(np.ascontiguousarray(rgb[:, :, c]), nw, nh) for c in range(3)])
    assert L.convert_in_memory(pil_png(rgb), p, FMT_JPEG) == O.write(O.forward(O.rgb_to_ycc(rz), op), op)


@pytest.mark.parametrize("name", ["in_420_base_355x237.jpg", "in_444_base_355x237.jpg", "in_gray_base_355x237.jpg", "in_420_prog_355x237.jpg"])
def test_convert_jpeg_to_lossless_png_matches_oracle_decode(L, O, golden, name):
    """JPEG -> PNG with png.optimize: the PNG must hold exactly the oracle's RGB decode of the JPEG (libjpeg-turbo-exact IDCT,
    fancy upsampling and colour conversion), also after a Lanczos3 resize."""
    from pngutil import pil_pixels
    data = golden(name)
    p = L.default_params(); p.png_optimize = 1; p.png_optimization_level = 2
    out = L.convert_in_memory(data, p, FMT_PNG)
    want = _jpeg_rgb(O, data)
    got = np.asarray(pil_pixels(out).convert("RGB")).transpose(2, 0, 1)
    assert np.array_equal(got, want)
    p.width = 120
    nw, nh = O.compute_dimensions(355, 237, 120, 0)
    got = np.asarray(pil_pixels(L.convert_in_memory(data, p, FMT_PNG)).convert("RGB")).transpose(2, 0, 1)
    assert np.array_equal(got, _jpeg_rgb(O, data, nw, nh))


def test_convert_refusals(L, golden):
    data = golden("in_420_base_355x237.jpg")
    p = L.default_params()
    for fmt, code in ((FMT_JPEG, 8), (FMT_PNG, 3), (FMT_GIF, 3)):
        with pytest.raises(L.B200Error) as e:
            L.convert_in_memory(data, p, fmt)
        assert e.value.code == code
    p.webp_lossless = 1
    with pytest.raises(L.B200Error) as e:
        L.convert_in_memory(data, p, FMT_WEBP)
    assert e.value.code == 3
    with pytest.raises(L.B200Error) as e:
        L.convert_in_memory(b"garbage", L.default_params(), FMT_WEBP)
    assert e.value.code == 2


def test_cli_format_webp_and_png_lossless(L, O, golden, tmp_path):
    """The b200clt mirror of caesiumclt drives the same entry points: --format webp (+ --width) and --lossless on a PNG."""
    import json
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "caesium-clt_b200", "b200clt")
    src = tmp_path / "in"; src.mkdir()
    (src / "a.jpg").write_bytes(golden("in_420_base_640x480.jpg"))
    (src / "b.png").write_bytes(pil_png(synth(64, 96, 3, seed=1)))
    out = tmp_path / "out"
    r = subprocess.run([exe, "-q", "85", "--width", "320", "--format", "webp", "-o", str(out), "--json", str(src / "a.jpg")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    p = L.default_params(); p.webp_quality = 85; p.jpeg_quality = 85; p.png_quality = 85; p.width = 320
    assert (out / "a.webp").read_bytes() == L.convert_in_memory(golden("in_420_base_640x480.jpg"), p, FMT_WEBP)
    json.loads(r.stdout)                                     # --json prints one valid document
    r = subprocess.run([exe, "--lossless", "-o", str(out), str(src / "b.png")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    from pngutil import pil_pixels
    assert np.array_equal(np.asarray(pil_pixels((out / "b.png").read_bytes())), np.asarray(pil_pixels((src / "b.png").read_bytes())))


def test_convert_full_size_config5_shape(L, O):
    """BASELINE configs[4] in miniature: a large JPEG, --width 1920 --format webp -q 85; file == oracle, decodes close to the
    Lanczos-resized source."""
    import io
    from PIL import Image
    img = synth(2000, 3000, 3, seed=3, kind="photo")
    b = io.BytesIO(); Image.fromarray(img).save(b, format="JPEG", quality=92, subsampling=2)
    p = L.default_params(); p.webp_quality = 85; p.width = 1920
    out = L.convert_in_memory(b.getvalue(), p, FMT_WEBP)
    nw, nh = O.compute_dimensions(3000, 2000, 1920, 0)
    rgb = _jpeg_rgb(O, b.getvalue(), nw, nh)
    assert out == O.webp_encode(rgb, 85)[0]
    dec = pil_decode(out)
    assert dec.shape == (nh, nw, 3) and np.abs(dec.astype(int) - rgb.transpose(1, 2, 0).astype(int)).mean() < 3.0


# ---- round 2: WebP input ----------------------------------------------------------------------------------------------------------
def _sample(name):
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_samples", name), "rb") as f:
        return f.read()


@pytest.mark.parametrize("name", ["w0.webp", "w1.webp"])
def test_compress_webp_input_matches_oracle(L, O, name):
    """caesium::compress_in_memory on a WebP (the reference's own samples): decode (host, == libwebp) -> K8 at webp.quality; the
    file is the oracle's encoding of libwebp's decode, also with a resize in between."""
    data = _sample(name)
    rgb = planar(pil_decode(data))
    for q in (80, 40):
        p = L.default_params(); p.webp_quality = q
        assert L.compress_in_memory(data, p) == O.webp_encode(rgb, q)[0], (name, q)
    p = L.default_params(); p.webp_quality = 75; p.width = 200
    nw, nh = O.compute_dimensions(rgb.shape[2], rgb.shape[1], 200, 0)
    want = O.webp_encode(np.stack([O.resize_plane(np.ascontiguousarray(rgb[c]), nw, nh) for c in range(3)]), 75)[0]
    assert L.compress_in_memory(data, p) == want


def test_convert_from_webp_and_compress_to_size(L, O):
    data = _sample("w0.webp")
    rgb = planar(pil_decode(data))
    # WebP -> JPEG: the PNG -> JPEG back end on the decoded pixels
    p = L.default_params(); p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = 80, 420, 1
    op = O.params(80, 420, True)
    assert L.convert_in_memory(data, p, FMT_JPEG) == O.write(O.forward(O.rgb_to_ycc(rgb), op), op)
    # WebP -> lossless PNG: holds exactly the decoded pixels
    from pngutil import pil_pixels
    p = L.default_params(); p.png_optimize = 1
    out = L.convert_in_memory(data, p, FMT_PNG)
    assert np.array_equal(np.asarray(pil_pixels(out).convert("RGB")).transpose(2, 0, 1), rgb)
    # compress_to_size on a WebP: quality bisection with the pixels resident on the device; the answer is the oracle's file at the
    # quality the call reports
    target = len(data) // 2
    p = L.default_params(); p.webp_quality = 80
    out = L.compress_to_size_in_memory(data, p, target)
    assert len(out) <= target and out[:4] == b"RIFF"
    assert out == O.webp_encode(rgb, int(p.webp_quality))[0]
    # the convert-then-size arm of the reference (compressor.rs:288-299): JPEG -> WebP, then to size
    src = _sample("j1.jpg")
    p = L.default_params(); p.webp_quality = 80; p.width = 400
    conv = L.convert_in_memory(src, p, FMT_WEBP)
    p2 = L.default_params(); p2.webp_quality = 80
    sized = L.compress_to_size_in_memory(conv, p2, len(conv) // 2)
    assert len(sized) <= len(conv) // 2 and pil_decode(sized).shape == pil_decode(conv).shape


def _chunks(f):
    assert f[:4] == b"RIFF" and f[8:12] == b"WEBP" and int.from_bytes(f[4:8], "little") == len(f) - 8
    out, pos = {}, 12
    while pos < len(f):
        n = int.from_bytes(f[pos + 4:pos + 8], "little")
        out[f[pos:pos + 4]] = f[pos + 8:pos + 8 + n]
        pos += 8 + n + (n & 1)
    return out


def _soft_alpha(h, w, seed):
    yy, xx = np.mgrid[:h, :w]
    a = np.clip(300 - np.hypot(yy - h / 2, xx - w / 2) * 600 / max(h, w), 0, 255).astype(np.uint8)
    a[: h // 8] = 0; a[:, : w // 10] = 255
    rng = np.random.default_rng(seed); a[h // 2:h // 2 + 4] = rng.integers(0, 256, (min(4, h - h // 2), w), dtype=np.uint8)
    return a


@pytest.mark.parametrize("h,w", [(90, 120), (1, 1), (257, 33), (600, 800)])
def test_convert_transparent_png_to_webp_keeps_the_alpha_plane(L, O, h, w):
    """PNG with real transparency -> VP8X file: the colour frame is the oracle's, the alpha plane is lossless (libwebp decodes it back
    exactly) and its ALPH chunk is the host coder's output for the ORACLE's LZ77 tokens of the plane (so K7's tokens == the twin's)."""
    import io
    from PIL import Image
    rgb, a = synth(h, w, 3, seed=h + w), _soft_alpha(h, w, 5)
    p = L.default_params(); p.webp_quality = 80
    out = L.convert_in_memory(pil_png(np.concatenate([rgb, a[:, :, None]], axis=2)), p, FMT_WEBP)
    ch = _chunks(out)
    assert set(ch) == {b"VP8X", b"ALPH", b"VP8 "} and ch[b"VP8X"][0] == 0x10
    assert int.from_bytes(ch[b"VP8X"][4:7], "little") == w - 1 and int.from_bytes(ch[b"VP8X"][7:10], "little") == h - 1
    assert ch[b"VP8 "] == _chunks(O.webp_encode(planar(rgb), 80)[0])[b"VP8 "]
    k, res = L.webp_alpha_filter(a)
    tok, _ = O.png_lz77(res.reshape(-1), 1, w)
    assert ch[b"ALPH"] == L.webp_alpha_chunk(tok, w, h, k)
    got = np.asarray(Image.open(io.BytesIO(out)).convert("RGBA"))
    assert np.array_equal(got[:, :, 3], a)
    assert np.array_equal(got[:, :, :3], pil_decode(O.webp_encode(planar(rgb), 80)[0]))


def test_convert_transparent_png_to_webp_with_resize_and_trns(L, O):
    import io
    from PIL import Image
    h, w = 240, 320
    rgb, a = synth(h, w, 3, seed=9), _soft_alpha(h, w, 6)
    p = L.default_params(); p.webp_quality = 75; p.width = 100
    out = L.convert_in_memory(pil_png(np.concatenate([rgb, a[:, :, None]], axis=2)), p, FMT_WEBP)
    nw, nh = O.compute_dimensions(w, h, 100, 0)
    got = np.asarray(Image.open(io.BytesIO(out)).convert("RGBA"))
    assert got.shape == (nh, nw, 4)
    assert np.array_equal(got[:, :, 3], O.resize_plane(a, nw, nh))            # the alpha plane takes the same Lanczos3 as the colour planes
    want_rgb = np.stack([O.resize_plane(rgb[:, :, c].copy(), nw, nh) for c in range(3)])
    assert _chunks(out)[b"VP8 "] == _chunks(O.webp_encode(want_rgb, 75)[0])[b"VP8 "]
    # an alpha channel that becomes opaque ... stays a simple file; a palette with tRNS carries per-entry alpha
    rng = np.random.default_rng(4)
    idx = rng.integers(0, 16, (40, 60)).astype(np.uint8)
    im = Image.fromarray(idx, mode="P"); im.putpalette([int(v) for v in rng.integers(0, 256, 48)])
    trns = bytes(int(v) for v in rng.integers(0, 256, 10))
    b = io.BytesIO(); im.save(b, "PNG", transparency=trns)
    p = L.default_params(); p.webp_quality = 80
    out = L.convert_in_memory(b.getvalue(), p, FMT_WEBP)
    got = np.asarray(Image.open(io.BytesIO(out)).convert("RGBA"))
    lut = np.full(256, 255, np.uint8); lut[:10] = np.frombuffer(trns, np.uint8)
    assert np.array_equal(got[:, :, 3], lut[idx])
    # colour key on a grey image
    g = rng.integers(0, 4, (30, 50)).astype(np.uint8) * 85
    b = io.BytesIO(); Image.fromarray(g, mode="L").save(b, "PNG", transparency=85)
    got = np.asarray(Image.open(io.BytesIO(L.convert_in_memory(b.getvalue(), p, FMT_WEBP))).convert("RGBA"))
    assert np.array_equal(got[:, :, 3], np.where(g == 85, 0, 255).astype(np.uint8))


def test_compress_webp_inputs_with_alpha_and_lossless(L, O):
    """WebP sources the VP8 decoder alone does not cover: a lossy file with an alpha plane is re-encoded with its alpha plane intact,
    a lossless (VP8L) file is decoded and re-encoded lossy; converted to PNG the transparency stays (RGBA); to JPEG it is dropped."""
    import io
    from PIL import Image
    from pngutil import pil_pixels
    h, w = 150, 210
    a = _soft_alpha(h, w, 3)
    img = np.concatenate([synth(h, w, 3, seed=12, kind="photo"), a[:, :, None]], axis=2)
    b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", quality=85, alpha_quality=100); lossy_alpha = b.getvalue()
    b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", lossless=True, exact=True); lossless_alpha = b.getvalue()
    b = io.BytesIO(); Image.fromarray(img[:, :, :3].copy()).save(b, "WEBP", lossless=True); lossless_rgb = b.getvalue()
    p = L.default_params(); p.webp_quality = 70
    for src in (lossy_alpha, lossless_alpha):
        dec = np.asarray(Image.open(io.BytesIO(src)).convert("RGBA"))
        out = L.compress_in_memory(src, p)
        ch = _chunks(out)
        assert set(ch) == {b"VP8X", b"ALPH", b"VP8 "}
        assert ch[b"VP8 "] == _chunks(O.webp_encode(planar(dec[:, :, :3]), 70)[0])[b"VP8 "]
        got = np.asarray(Image.open(io.BytesIO(out)).convert("RGBA"))
        assert np.array_equal(got[:, :, 3], dec[:, :, 3])
        # -> PNG keeps the transparency, -> JPEG drops it
        pp = L.default_params(); pp.png_optimize = 1
        png = np.asarray(pil_pixels(L.convert_in_memory(src, pp, FMT_PNG)).convert("RGBA"))
        assert np.array_equal(png, dec)
        pj = L.default_params(); pj.jpeg_quality, pj.jpeg_chroma_subsampling, pj.jpeg_progressive = 80, 420, 1
        op = O.params(80, 420, True)
        assert L.convert_in_memory(src, pj, FMT_JPEG) == O.write(O.forward(O.rgb_to_ycc(planar(dec[:, :, :3])), op), op)
    dec = np.asarray(Image.open(io.BytesIO(lossless_rgb)).convert("RGB"))
    assert L.compress_in_memory(lossless_rgb, p) == O.webp_encode(planar(dec), 70)[0]
    # resized: colour and alpha planes take the same Lanczos3
    p.width = 100
    nw, nh = O.compute_dimensions(w, h, 100, 0)
    dec = np.asarray(Image.open(io.BytesIO(lossy_alpha)).convert("RGBA"))
    got = np.asarray(Image.open(io.BytesIO(L.compress_in_memory(lossy_alpha, p))).convert("RGBA"))
    assert np.array_equal(got[:, :, 3], O.resize_plane(np.ascontiguousarray(dec[:, :, 3]), nw, nh))
    pp = L.default_params(); pp.png_optimize = 1; pp.width = 100
    png = np.asarray(pil_pixels(L.convert_in_memory(lossy_alpha, pp, FMT_PNG)).convert("RGBA"))
    assert np.array_equal(png[:, :, 3], O.resize_plane(np.ascontiguousarray(dec[:, :, 3]), nw, nh))
    assert np.array_equal(png[:, :, 0], O.resize_plane(np.ascontiguousarray(dec[:, :, 0]), nw, nh))


def test_convert_webp_to_png_with_resize_matches_oracle(L, O):
    """WebP -> lossless PNG at width=100, for an opaque file and one with an alpha plane: every channel of the PNG is the oracle's
    Lanczos3 of the decoded source's channel."""
    import io
    from PIL import Image
    from pngutil import pil_pixels
    h, w = 150, 210
    img = np.concatenate([synth(h, w, 3, seed=12, kind="photo"), _soft_alpha(h, w, 3)[:, :, None]], axis=2)
    b = io.BytesIO(); Image.fromarray(img).save(b, "WEBP", quality=85, alpha_quality=100); lossy_alpha = b.getvalue()
    p = L.default_params(); p.png_optimize = 1; p.width = 100
    for src, mode in ((_sample("w0.webp"), "RGB"), (lossy_alpha, "RGBA")):
        dec = np.asarray(Image.open(io.BytesIO(src)).convert(mode))
        nw, nh = O.compute_dimensions(dec.shape[1], dec.shape[0], 100, 0)
        png = np.asarray(pil_pixels(L.convert_in_memory(src, p, FMT_PNG)).convert(mode))
        assert png.shape == (nh, nw, len(mode)), mode
        for c in range(len(mode)):
            assert np.array_equal(png[:, :, c], O.resize_plane(np.ascontiguousarray(dec[:, :, c]), nw, nh)), (mode, c)
