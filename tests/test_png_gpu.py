"""GPU parity tests of the lossless PNG leg (SURVEY.md §8 row a8): K6 row filtering and K7 LZ77 against the oracle
(bit-exact filter choices, filtered bytes, tokens and histograms), and the whole b200_compress_in_memory PNG path against
the one property that defines it -- the output decodes (libpng via Pillow) to exactly the input's pixels."""
import io
import zlib

import numpy as np
import pytest

from pngutil import idat_stream, pil_pixels, pil_png, synth

pytestmark = pytest.mark.gpu


def lossless_params(L, level=3, keep_metadata=False):
    p = L.default_params()
    p.png_optimize = 1
    p.png_optimization_level = level
    p.keep_metadata = 1 if keep_metadata else 0
    return p


@pytest.mark.parametrize("shape", [(37, 53), (1, 1), (3, 700), (130, 9), (64, 1024)])
@pytest.mark.parametrize("channels", [1, 2, 3, 4])
def test_filter_kernel_matches_oracle(L, O, shape, channels):
    h, w = shape
    for kind in ("photo", "flat"):
        raw = synth(h, w, channels, seed=h + w + channels, kind=kind).reshape(h, w * channels)
        for s in range(10):
            got = L.png_filter(raw, channels, s)
            want = O.png_filter(raw, channels, s)
            assert np.array_equal(got[:, 0], want[:, 0]), (kind, s, "filter choice")
            assert np.array_equal(got, want), (kind, s)


def test_filter_kernel_16bit_and_subbyte_rows(L, O):
    rng = np.random.default_rng(1)
    raw = rng.integers(0, 256, (40, 2 * 3 * 31)).astype(np.uint8)         # 16-bit RGB: bpp 6
    for s in range(10):
        assert np.array_equal(L.png_filter(raw, 6, s), O.png_filter(raw, 6, s))
    raw = rng.integers(0, 256, (40, 13)).astype(np.uint8)                 # packed 1/2/4-bit rows: bpp 1
    for s in range(10):
        assert np.array_equal(L.png_filter(raw, 1, s), O.png_filter(raw, 1, s))


@pytest.mark.parametrize("kind,channels,shape", [("photo", 3, (64, 97)), ("flat", 3, (200, 333)), ("flat", 1, (100, 4100)), ("noise", 4, (50, 50)),
                                                  ("photo", 2, (31, 17)), ("flat", 4, (1, 5)), ("flat", 1, (1, 2))])
def test_lz77_kernels_match_oracle(L, O, kind, channels, shape):
    h, w = shape
    img = synth(h, w, channels, seed=3, kind=kind)
    filt = O.png_filter(img.reshape(h, -1), channels, 4 if kind == "photo" else 0)
    stream = filt.reshape(-1)
    tok, hist = L.png_lz77(stream, channels, filt.shape[1])
    wtok, whist = O.png_lz77(stream, channels, filt.shape[1])
    assert np.array_equal(hist, whist)
    assert np.array_equal(tok, wtok)
    assert np.array_equal(O.png_expand(tok, stream.size), stream)


def _check_lossless(L, png_in, level=3, expect_mode=None):
    out = L.compress_in_memory(png_in, lossless_params(L, level))
    a, b = pil_pixels(png_in), pil_pixels(out)
    assert a.size == b.size
    if expect_mode:
        assert b.mode == expect_mode
    if a.mode != b.mode:                      # a colour-type reduction: compare in the richer mode
        b = b.convert(a.mode)
    assert np.array_equal(np.asarray(a), np.asarray(b))
    ihdr, idat, order = idat_stream(out)
    assert order[0] == b"IHDR" and order[-1] == b"IEND"
    filt = zlib.decompress(idat)              # a complete, valid zlib stream with a correct Adler-32
    return out, ihdr, filt


@pytest.mark.parametrize("level", [0, 1, 2, 3, 5, 6])
def test_compress_png_is_lossless_at_every_level(L, level):
    img = synth(120, 160, 3, seed=level, kind="photo")
    out, ihdr, filt = _check_lossless(L, pil_png(img), level)
    assert len(filt) == 120 * (160 * 3 + 1)
    if level == 0:
        assert set(filt[::160 * 3 + 1]) == {0}


@pytest.mark.parametrize("channels,kind", [(1, "photo"), (2, "photo"), (3, "flat"), (4, "photo"), (4, "flat")])
def test_compress_png_colour_types(L, channels, kind):
    _check_lossless(L, pil_png(synth(77, 131, channels, seed=channels, kind=kind)))


def test_compress_png_smaller_than_a_naive_encoder(L):
    img = synth(256, 256, 3, seed=8, kind="photo")
    src = pil_png(img, compress_level=1)
    out, _, _ = _check_lossless(L, src)
    assert len(out) < len(src)
    flat = synth(256, 256, 3, seed=8, kind="flat")
    out2, _, _ = _check_lossless(L, pil_png(flat, compress_level=1))
    assert len(out2) < 256 * 256 * 3 // 20


def test_compress_png_reductions(L):
    rgb = synth(60, 80, 3, seed=1)
    opaque = np.concatenate([rgb, np.full((60, 80, 1), 255, np.uint8)], axis=2)
    _check_lossless(L, pil_png(opaque), expect_mode="RGB")                   # opaque alpha dropped
    grey3 = np.repeat(synth(60, 80, 1, seed=2), 3, axis=2)
    _check_lossless(L, pil_png(grey3), expect_mode="L")                      # r == g == b -> greyscale
    grey4 = np.concatenate([grey3, synth(60, 80, 1, seed=5)], axis=2)
    _check_lossless(L, pil_png(grey4), expect_mode="LA")                     # grey + real alpha
    both = np.concatenate([grey3, np.full((60, 80, 1), 255, np.uint8)], axis=2)
    _check_lossless(L, pil_png(both), expect_mode="L")
    real = np.concatenate([rgb, synth(60, 80, 1, seed=6)], axis=2)
    _check_lossless(L, pil_png(real), expect_mode="RGBA")                    # nothing to reduce


def test_compress_png_palette_reduction(L):
    """<= 256 colours: the file comes back indexed (PLTE + tRNS), pixel-exact, and far smaller than one byte per sample"""
    for ch in (3, 4):
        img = synth(150, 220, ch, seed=40 + ch, kind="flat")
        if ch == 4:
            img[20:60, 30:90, 3] = 0; img[100:110, :, 3] = 77
        out, ihdr, filt = _check_lossless(L, pil_png(img), expect_mode="P")
        n = len(np.unique(img.reshape(-1, ch), axis=0))
        depth = 1 if n <= 2 else 2 if n <= 4 else 4 if n <= 16 else 8
        assert ihdr[2] == depth and ihdr[3] == 3 and len(filt) == 150 * ((220 * depth + 7) // 8 + 1)
        assert len(out) < 150 * 220 // 8


def test_compress_png_palette_16bit_and_bilevel(L):
    from PIL import Image
    rng = np.random.default_rng(3)
    idx = (synth(50, 70, 1, seed=3, kind="flat")[:, :, 0] % 16).astype(np.uint8)
    im = Image.fromarray(idx, mode="P"); im.putpalette([int(v) for v in rng.integers(0, 256, 48)])
    src = pil_png(im)
    out = L.compress_in_memory(src, lossless_params(L))
    assert np.array_equal(np.asarray(pil_pixels(src).convert("RGB")), np.asarray(pil_pixels(out).convert("RGB")))
    a16 = (synth(40, 40, 1, seed=4)[:, :, 0].astype(np.uint16) * 257) ^ 0x0103
    src = pil_png(Image.fromarray(a16))
    out = L.compress_in_memory(src, lossless_params(L))
    assert np.array_equal(np.asarray(pil_pixels(src)), np.asarray(pil_pixels(out)))
    bw = rng.integers(0, 2, (33, 47)).astype(bool)
    src = pil_png(Image.fromarray(bw))
    out = L.compress_in_memory(src, lossless_params(L))
    assert np.array_equal(np.asarray(pil_pixels(src)), np.asarray(pil_pixels(out)))


def test_compress_png_transparency_chunk_survives(L):
    from PIL import Image
    idx = (synth(20, 20, 1, seed=3, kind="flat")[:, :, 0] % 4).astype(np.uint8)
    im = Image.fromarray(idx, mode="P"); im.putpalette([0, 0, 0, 255, 0, 0, 0, 255, 0, 0, 0, 255])
    b = io.BytesIO(); im.save(b, format="PNG", transparency=bytes([0, 128, 255, 255]))
    out = L.compress_in_memory(b.getvalue(), lossless_params(L))
    assert np.array_equal(np.asarray(pil_pixels(b.getvalue()).convert("RGBA")), np.asarray(pil_pixels(out).convert("RGBA")))


def test_compress_png_metadata_policy(L):
    from PIL import Image
    from PIL.PngImagePlugin import PngInfo
    meta = PngInfo(); meta.add_text("Comment", "hello from the test")
    b = io.BytesIO(); Image.fromarray(synth(16, 16, 3)).save(b, format="PNG", pnginfo=meta, dpi=(300, 300))
    _, _, kept = idat_stream(L.compress_in_memory(b.getvalue(), lossless_params(L, keep_metadata=True)))
    _, _, stripped = idat_stream(L.compress_in_memory(b.getvalue(), lossless_params(L, keep_metadata=False)))
    assert b"tEXt" in kept and b"tEXt" not in stripped
    assert b"pHYs" in kept and b"pHYs" in stripped          # oxipng StripChunks::Safe keeps pHYs


def test_compress_png_large_image(L):
    img = synth(1080, 1920, 3, seed=2, kind="photo")
    src = pil_png(img, compress_level=1)
    out, _, filt = _check_lossless(L, src)
    assert len(filt) == 1080 * (1920 * 3 + 1) and len(out) < len(src)


def test_png_paths_outside_the_gpu_build_are_refused(L):
    src = pil_png(synth(16, 16, 3))
    p = L.default_params(); p.png_optimize = 0                      # lossy = imagequant
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(src, p)
    assert e.value.code == 3
    p = lossless_params(L); p.width = 8
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(src, p)
    assert e.value.code == 3
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(src[:50], lossless_params(L))
    assert e.value.code == 4


def test_compress_batch_mixes_png_and_jpeg(L, golden):
    items = [pil_png(synth(64, 64, 3, seed=i)) for i in range(3)] + [golden("in_420_base_355x237.jpg")]
    p = lossless_params(L)
    outs = L.compress_batch(items, p)
    for src, (data, code, msg) in zip(items, outs):
        assert code == 0, msg
        if src[:2] == b"\xff\xd8":
            assert data[:2] == b"\xff\xd8"
        else:
            assert np.array_equal(np.asarray(pil_pixels(src)), np.asarray(pil_pixels(data)))


# ---- round 2: un-filtering, checksum verification and DEFLATE coding moved to the device -------------------------------------------
def _mixed_filter_png(O, img, bit_depth=8, seed=0):
    """A PNG whose rows use random filter types 0..4 (oracle filters, framed by zlib): every reconstruction branch of the wavefront."""
    h = img.shape[0]
    raw = img.reshape(h, -1)
    ch = {1: 0, 2: 4, 3: 2, 4: 6}[img.shape[2] // (bit_depth // 8 if bit_depth >= 8 else 1)] if bit_depth >= 8 else 0
    bpp = max(1, img.shape[2]) if bit_depth >= 8 else 1
    per = [O.png_filter(raw, bpp, s) for s in range(5)]
    rng = np.random.default_rng(seed)
    pick = rng.integers(0, 5, h)
    rows = np.stack([per[pick[y]][y] for y in range(h)])
    from pngutil import frame_png
    width = img.shape[1] if bit_depth >= 8 else img.shape[1] * 8 // bit_depth
    return frame_png(width, h, bit_depth, ch, zlib.compress(rows.tobytes(), 6)), pick


@pytest.mark.parametrize("shape,channels,depth", [((67, 131), 3, 8), ((200, 97), 4, 8), ((33, 500), 1, 8), ((90, 64), 2, 8), ((40, 70), 6, 16), ((35, 45), 8, 16),
                                                   ((129, 33), 3, 8), ((1, 1), 4, 8), ((32, 1), 3, 8), ((31, 2), 1, 8), ((64, 40), 1, 2)])
def test_device_unfilter_every_filter_type_and_pixel_size(L, O, shape, channels, depth):
    h, w = shape
    rng = np.random.default_rng(h * w + channels)
    img = rng.integers(0, 256, (h, w, channels)).astype(np.uint8)
    # smooth-ish content so that Paeth / Average predictions matter
    img = (img // 8 + (np.add.outer(np.arange(h), np.arange(w))[:, :, None] * 3) % 200).astype(np.uint8)
    src, pick = _mixed_filter_png(O, img, depth, seed=h)
    assert len(set(pick.tolist())) >= min(5, h) or h < 5
    out = L.compress_in_memory(src, lossless_params(L, 2))
    a, b = pil_pixels(src), pil_pixels(out)
    assert a.size == b.size
    conv = "RGBA" if a.mode in ("RGBA", "LA", "P") or b.mode in ("RGBA", "LA", "P") else a.mode
    if depth == 16 or a.mode.startswith("I"):
        assert np.array_equal(np.asarray(a), np.asarray(b))
    else:
        assert np.array_equal(np.asarray(a.convert(conv)), np.asarray(b.convert(conv)))


def test_device_checks_of_the_input_stream(L, O):
    """Adler-32 of the inflated IDAT is verified on the device; a filter byte > 4 is refused: both are corrupt input (code 4)."""
    from pngutil import frame_png
    img = synth(40, 50, 3, seed=4)
    rows = O.png_filter(img.reshape(40, -1), 3, 4)
    z = bytearray(zlib.compress(rows.tobytes(), 6))
    z[-1] ^= 0x55                                                   # break the stored Adler-32 only
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(frame_png(50, 40, 8, 2, bytes(z)), lossless_params(L))
    assert e.value.code == 4 and "Adler" in str(e.value)
    bad = rows.copy(); bad[7, 0] = 9
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(frame_png(50, 40, 8, 2, zlib.compress(bad.tobytes(), 6)), lossless_params(L))
    assert e.value.code == 4 and "filter" in str(e.value)
    assert L.compress_in_memory(frame_png(50, 40, 8, 2, zlib.compress(rows.tobytes(), 6)), lossless_params(L))[:4] == b"\x89PNG"


@pytest.mark.parametrize("kind,shape", [("photo", (300, 400)), ("flat", (257, 300)), ("noise", (120, 90)), ("photo", (1, 3))])
def test_device_deflate_writer_equals_host_writer(L, O, kind, shape):
    """The zlib stream the device writes (k_dfl_*: per-block statistics, code lengths, header, bit packing) is bit for bit the
    stream the host writer (deflate_tokens, the same dfl_core.h bodies run sequentially) makes from the same tokens."""
    h, w = shape
    img = synth(h, w, 3, seed=h + w, kind=kind)
    src = pil_png(img, compress_level=1)
    out = L.compress_in_memory(src, lossless_params(L, 3))
    ihdr, idat, _ = idat_stream(out)
    filt = np.frombuffer(zlib.decompress(idat), np.uint8)
    channels = {2: 3, 6: 4, 0: 1, 4: 2, 3: 1}[ihdr[3]]
    # a palette-reduced image (few colours) is coded from its indexed rows, possibly packed below a byte per pixel
    bpp = max(1, channels * ihdr[2] // 8)
    stride = filt.size // h
    tok, _ = L.png_lz77(filt, bpp, stride)
    want = L.png_deflate_tokens(tok, zlib.adler32(filt.tobytes()))
    assert idat == want
