"""PNG -> PNG with a target size on the device (b200_set_png_resize): the stage entry against the oracle twin byte for byte, and
every call that reaches the leg -- lossless, lossy, compress_to_size, batch, the CLI -- decoding to the twin's resized samples."""
import os
import struct
import subprocess
import sys
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import png_resize_cases as cases
from oracle import png_resize as R
from pngutil import chunk, frame_png, idat_stream, pil_pixels, pil_png, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def rz(L):
    assert L.set_png_resize(True) == 0
    yield L
    L.set_png_resize(False)


@pytest.fixture
def both(rz):
    assert rz.set_png_lossy(True) == 0
    yield rz
    rz.set_png_lossy(False)


# (source w, h) -> (width, height) as in b200_params
SHAPES = [((1, 1), (0, 0)), ((1, 1), (1, 1)), ((1, 17), (1, 40)), ((23, 1), (9, 1)), ((37, 53), (13, 0)), ((64, 1024), (0, 100)),
          ((9, 7), (40, 0)), ((30, 20), (45, 7))]


def oracle_of(O, c, dw, dh):
    return R.png_resize(c["raw"], c["width"], c["height"], c["bit_depth"], c["color_type"], c["plte"], c["trns"], dw, dh)


@pytest.mark.parametrize("ct,bd,trns", cases.LEGAL, ids=[cases.case_id(*k) for k in cases.LEGAL])
def test_stage_entry_equals_the_oracle(L, O, ct, bd, trns):
    for (w, h), (dw, dh) in SHAPES:
        c = cases.make(O, ct, bd, trns, w, h, seed=w * 7 + h)
        info, rows = L.png_resize_samples(c["png"], dw, dh)
        want, wrows = oracle_of(O, c, dw, dh)
        assert (info.width, info.height, info.bit_depth, info.color_type, info.row_bytes) == \
            (want["width"], want["height"], want["bit_depth"], want["color_type"], want["row_bytes"]), ((w, h), (dw, dh))
        assert info.bpp == want["channels"] * want["bit_depth"] // 8
        assert np.array_equal(rows, wrows), ((w, h), (dw, dh))


def _chunks(png):
    pos, out = 8, []
    while pos < len(png):
        n, tag = struct.unpack(">I4s", png[pos:pos + 8])
        out.append((tag, png[pos + 8:pos + 8 + n]))
        pos += 12 + n
    return out


def _rgba(planes, depth):
    """planes of any decoded type -> [h, w, 4] at that depth (grey replicated, missing alpha at the maximum)"""
    top = 65535 if depth == 16 else 255
    p = planes.astype(np.int64)
    if p.shape[0] in (1, 2):
        p = np.concatenate([p[:1], p[:1], p[:1], p[1:]], 0)
    if p.shape[0] == 3:
        p = np.concatenate([p, np.full((1,) + p.shape[1:], top)], 0)
    return np.moveaxis(p, 0, -1)


def decode_exact(O, png):
    """a PNG file -> ([h, w, 4] int64 samples at its own depth, depth): zlib checked, un-filtered by the oracle, expanded"""
    ch = dict(_chunks(png))
    w, h, bd, ct = struct.unpack(">IIBB", ch[b"IHDR"][:10])
    _, idat, _ = idat_stream(png)
    filt = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, -1)
    bpp = max(1, cases.NIN[ct] * bd // 8)
    raw = O.png_unfilter(filt, bpp)
    planes = R.expand_planes(raw, w, h, bd, ct, ch.get(b"PLTE", b""), ch.get(b"tRNS", b""))
    return _rgba(planes, 16 if bd == 16 else 8), (w, h)


def want_rgba(info, rows):
    planes = R.expand_planes(rows, info["width"], info["height"], info["bit_depth"], info["color_type"])
    return _rgba(planes, info["bit_depth"])


def params(L, width=0, height=0, level=3, optimize=1, q=80):
    p = L.default_params()
    p.png_optimize, p.png_optimization_level, p.png_quality, p.width, p.height = optimize, level, q, width, height
    return p


LOSSLESS = [(2, 8, False), (6, 8, False), (0, 16, True), (2, 16, False), (3, 2, True), (3, 8, False), (0, 4, False), (4, 8, False)]


@pytest.mark.parametrize("level", [0, 3, 6])
def test_lossless_decodes_to_the_oracle(rz, O, level):
    for ct, bd, trns in LOSSLESS:
        for (w, h), (dw, dh) in [((37, 53), (13, 0)), ((9, 7), (40, 0)), ((30, 20), (45, 7)), ((24, 18), (24, 18))]:
            c = cases.make(O, ct, bd, trns, w, h, seed=ct + bd + w)
            out = rz.compress_in_memory(c["png"], params(rz, dw, dh, level))
            info, rows = oracle_of(O, c, dw, dh)
            got, size = decode_exact(O, out)
            assert size == (info["width"], info["height"]) == O.compute_dimensions(w, h, dw, dh)
            assert np.array_equal(got, want_rgba(info, rows)), (ct, bd, trns, (w, h), (dw, dh))


def test_a_flat_image_resized_is_reduced_to_a_palette(rz, O):
    img = np.zeros((40, 60, 3), np.uint8)
    img[:, 30:] = (200, 10, 40)
    out = rz.compress_in_memory(pil_png(img), params(rz, 60, 40))      # same size: expanded, not resampled, then reduced
    assert any(t == b"PLTE" for t, _ in _chunks(out))
    assert np.array_equal(np.asarray(pil_pixels(out).convert("RGB")), img)


@pytest.mark.parametrize("q", [40, 80])
def test_lossy_decodes_to_the_quantiser_twin(both, O, q):
    for ct, bd, trns in [(6, 8, False), (2, 16, False), (0, 8, True), (3, 4, True)]:
        c = cases.make(O, ct, bd, trns, 48, 36, seed=q + ct)
        out = both.compress_in_memory(c["png"], params(both, 31, 0, optimize=0, q=q))
        info, rows = oracle_of(O, c, 31, 0)
        got = np.asarray(pil_pixels(out).convert("RGBA"))
        assert np.array_equal(got, R.quantized_rgba(info, rows, q)), (ct, bd, trns)


def test_lossy_needs_the_lossy_switch(rz, O):
    c = cases.make(O, 2, 8, False, 20, 20)
    with pytest.raises(rz.B200Error) as e:
        rz.compress_in_memory(c["png"], params(rz, 10, 0, optimize=0))
    assert e.value.code == 3 and "lossy PNG" in str(e.value)


def test_compress_to_size_with_resize(both):
    L = both
    src = pil_png(synth(120, 160, 3, seed=11))
    small, big = (len(L.compress_in_memory(src, params(L, 100, 0, optimize=0, q=q))) for q in (1, 100))
    limit = (small + big) // 2
    p = params(L, 100, 0, optimize=0, q=80)
    out = L.compress_to_size_in_memory(src, p, limit)
    assert len(out) <= limit
    assert out == L.compress_in_memory(src, params(L, 100, 0, optimize=0, q=p.png_quality))
    assert struct.unpack(">II", dict(_chunks(out))[b"IHDR"][:8]) == (100, 75)


def test_batch_and_threads_equal_single_calls(rz, O, golden):
    L = rz
    srcs = [cases.make(O, ct, bd, t, 50 + 9 * i, 41, seed=i)["png"] for i, (ct, bd, t) in enumerate(LOSSLESS[:5])]
    srcs.append(golden("in_420_base_355x237.jpg"))
    p = params(L, 33, 0)
    res = L.compress_batch(srcs, p, n_threads=3)
    singles = [L.compress_in_memory(s, p) for s in srcs]
    for (data, code, msg), single in zip(res, singles):
        assert code == 0, msg
        assert data == single
    with ThreadPoolExecutor(4) as ex:
        outs = list(ex.map(lambda s: L.compress_in_memory(s, p), [srcs[1]] * 8))
    assert all(o == singles[1] for o in outs)


def test_switch_off_still_refuses(L, O):
    L.set_png_resize(False)
    src = cases.make(O, 2, 8, False, 20, 20)["png"]
    L.set_png_lossy(True)
    try:
        for call in (lambda: L.compress_in_memory(src, params(L, 10)), lambda: L.compress_to_size_in_memory(src, params(L, 10, optimize=0), 10)):
            with pytest.raises(L.B200Error) as e:
                call()
            assert e.value.code == 3 and "PNG resize is outside the GPU path" in str(e.value)
    finally:
        L.set_png_lossy(False)
    (data, code, msg), = L.compress_batch([src], params(L, 10), n_threads=1)
    assert code == 3 and "PNG resize" in msg
    assert L.lib().b200_set_png_resize(2) != 0


_CHILD = """
import sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
from conftest import _import_pkg
_import_pkg()
import caesium_clt_b200._lib as L
from pngutil import pil_png, synth
p = L.default_params(); p.png_optimize = 1; p.width = 12
out = L.compress_in_memory(pil_png(synth(20, 24, 3)), p)
import struct
print(struct.unpack(">II", out[16:24]))
"""


def test_environment_variable_turns_the_switch_on():
    env = dict(os.environ, B200_PNG_RESIZE="gpu")
    r = subprocess.run([sys.executable, "-c", _CHILD.format(tests=os.path.join(ROOT, "tests"), root=ROOT)], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == "(12, 10)"


def test_cli_resizes_with_the_variable_and_refuses_without(tmp_path):
    src = tmp_path / "in" / "some.png"
    src.parent.mkdir()
    src.write_bytes(pil_png(synth(90, 120, 3, seed=5)))
    exe = os.path.join(ROOT, "caesium-clt_b200", "b200clt")
    out = tmp_path / "out"
    env = dict(os.environ, B200_PNG_RESIZE="gpu")
    r = subprocess.run([exe, "--lossless", "--width", "64", "-o", str(out), str(src)], env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert struct.unpack(">II", (out / "some.png").read_bytes()[16:24]) == (64, 48)
    env.pop("B200_PNG_RESIZE")
    out2 = tmp_path / "out2"
    r = subprocess.run([exe, "--lossless", "--width", "64", "-o", str(out2), str(src)], env=env, capture_output=True, text=True)
    assert "PNG resize is outside the GPU path" in r.stdout + r.stderr


def _corrupt_sources():
    img = synth(20, 30, 3, seed=3)
    rows = b"".join(b"\x01" + img[y].tobytes() for y in range(20))
    z = zlib.compress(rows)
    stride = 1 + 30 * 3
    bad_filter = zlib.compress(rows[:stride * 3] + b"\x07" + rows[stride * 3 + 1:])       # row 3's filter type
    bad_adler = z[:-4] + bytes(b ^ 0x5A for b in z[-4:])
    return {"truncated_idat": frame_png(30, 20, 8, 2, z[: len(z) // 2]), "bad_filter": frame_png(30, 20, 8, 2, bad_filter),
            "adler": frame_png(30, 20, 8, 2, bad_adler)}


@pytest.mark.parametrize("which", ["truncated_idat", "bad_filter", "adler"])
def test_corrupt_input_is_code_4(both, which):
    src = _corrupt_sources()[which]
    for p in (params(both, 13), params(both, 13, optimize=0)):
        with pytest.raises(both.B200Error) as e:
            both.compress_in_memory(src, p)
        assert e.value.code == 4, str(e.value)
    with pytest.raises(both.B200Error) as e:
        both.png_resize_samples(src, 13, 0)
    assert e.value.code == 4


def test_resized_output_carries_no_source_chunks(both, O):
    img = synth(30, 40, 3, seed=8)
    rows = b"".join(b"\x00" + img[y].tobytes() for y in range(30))
    extra = chunk(b"sBIT", b"\x08\x08\x08") + chunk(b"pHYs", struct.pack(">IIB", 2835, 2835, 1)) + chunk(b"bKGD", struct.pack(">HHH", 1, 2, 3)) + \
        chunk(b"tEXt", b"Comment\x00kept?")
    src = frame_png(40, 30, 8, 2, zlib.compress(rows), extra)
    keep = params(both, 20); keep.keep_metadata = 1
    ref = both.compress_in_memory(src, params(both, 20))
    for p in (keep, params(both, 20, optimize=0)):
        p.keep_metadata = 1
        tags = [t for t, _ in _chunks(both.compress_in_memory(src, p))]
        assert set(tags) <= {b"IHDR", b"PLTE", b"tRNS", b"IDAT", b"IEND"}, tags
    assert both.compress_in_memory(src, keep) == ref
    p = params(both, 0); p.keep_metadata = 1; p.width = p.height = 0                 # without a resize the chunks stay
    assert b"tEXt" in [t for t, _ in _chunks(both.compress_in_memory(src, p))]


def _rgb16_photo(h, w, seed):
    img = synth(h, w, 3, seed=seed).astype(np.uint16) * 257 + (np.arange(h * w * 3).reshape(h, w, 3) % 199).astype(np.uint16)
    rows = b"".join(b"\x00" + img[y].astype(">u2").tobytes() for y in range(h))
    return frame_png(w, h, 16, 2, zlib.compress(rows, 1)), img


def test_real_sizes_equal_the_oracle(rz, O):
    yy, xx = np.mgrid[:4096, :4096]
    a = np.clip(300 - np.hypot(yy - 2048, xx - 2048) * 600 / 4096, 0, 255).astype(np.uint8)
    rgba = np.concatenate([synth(4096, 4096, 3, seed=1), a[:, :, None]], 2)
    png16, img16 = _rgb16_photo(1500, 2000, 2)
    for src, (w, h, bd, ct), raw in ((pil_png(rgba, compress_level=1), (4096, 4096, 8, 6), rgba.reshape(4096, -1)),
                                     (png16, (2000, 1500, 16, 2), img16.astype(">u2").view(np.uint8).reshape(1500, -1))):
        info, rows = rz.png_resize_samples(src, 1920, 0)
        want, wrows = R.png_resize(raw, w, h, bd, ct, b"", b"", 1920, 0)
        assert (info.width, info.height) == (want["width"], want["height"]) == ((1920, 1920) if w == h else (1920, 1440))
        assert np.array_equal(rows, wrows)
        out = rz.compress_in_memory(src, params(rz, 1920, 0, level=1))
        got, _ = decode_exact(O, out)
        assert np.array_equal(got, want_rgba(want, wrows))
