"""The GIF leg on the CPU: the host decoder (b200_gif_decode) against the independent reader tests/gifutil.py, that reader against
Pillow, refusals of malformed files, the LZW walk of gif_core.h (compiled for the CPU) decoding back to its input around segment
boundaries, and the oracle twin's files as a viewer shows them."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

import gif_cases
import gifutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
GIF_SEG = 16384

CASES = gif_cases.cases()
IDS = [n for n, _ in CASES]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libgif_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gif_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "gif_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emul_gif_lzw.restype = C.c_longlong
    return lib


def emul_lzw(emul, idx, m, seg):
    idx = np.ascontiguousarray(idx, np.uint8)
    cap = 64 + 2 * idx.size
    out = np.zeros(cap, np.uint8)
    n = emul.emul_gif_lzw(idx.ctypes.data_as(C.c_void_p), C.c_size_t(idx.size), int(m), int(seg), out.ctypes.data_as(C.c_void_p), C.c_size_t(cap))
    assert n > 0
    return out[:n].tobytes()


def unblock(data):
    body, end = gifutil._blocks(data, 0)
    assert end == len(data)
    return body


@pytest.mark.parametrize("name,data", CASES, ids=IDS)
def test_decoder_matches_independent_reader(L, name, data):
    canv, delays, loop = L.gif_decode(data)
    frames, loop_ref = gifutil.decode(data)
    assert len(canv) == len(frames)
    for k, (c, (ref, d)) in enumerate(zip(canv, frames)):
        assert np.array_equal(c, ref), (name, k)
        assert delays[k] == d
    assert loop == loop_ref
    assert set(np.unique(canv[..., 3])) <= {0, 255}
    assert not np.any(canv[canv[..., 3] == 0])


@pytest.mark.parametrize("name,data", [c for c in CASES if c[0].startswith(("still", "noise", "anim_opaque", "g1"))], ids=lambda v: v if isinstance(v, str) else "")
def test_independent_reader_matches_pillow(name, data):
    frames, loop = gifutil.decode(data)
    im = Image.open(io.BytesIO(data))
    assert im.n_frames == len(frames)
    for k, (canvas, delay) in enumerate(frames):
        im.seek(k)
        ref = np.asarray(im.convert("RGBA"))
        opaque = canvas[..., 3] == 255
        assert np.array_equal(canvas[opaque], ref[opaque]), (name, k)
        assert np.all(ref[~opaque][:, 3] == 0)
        assert delay == im.info.get("duration", 0) // 10
    assert loop == im.info.get("loop")


def test_minimum_code_sizes_two_to_eight():
    seen = {gifutil.parse(data)["frames"][0]["min_code_size"] for name, data in CASES if name.startswith("still_m")}
    assert seen == set(range(2, 9))


def test_pillow_stream_fills_the_dictionary():
    info = gifutil.parse(dict(CASES)["noise"])
    f = info["frames"][0]
    assert f["w"] * f["h"] > 4096 * 4


def _mutations(data):
    d = bytearray(data)
    yield "empty screen", bytes(d[:6] + b"\x00\x00" + d[8:])
    for cut in (5, 12, 13, len(d) // 3, len(d) // 2, len(d) - 2, len(d) - 1):
        yield "truncated at %d" % cut, bytes(d[:cut])
    i = d.index(b"\x2c")
    bad = bytearray(d)
    bad[i + 10 + (3 * (2 << (d[10] & 7)) if d[i + 9] & 0x80 else 0)] = 12
    yield "min code size 12", bytes(bad)
    yield "no trailer", bytes(d[:-1]) + b"\x00"
    yield "unknown block", bytes(d[:-1]) + b"\x99"
    yield "no frames", bytes(d[:13 + (3 * (2 << (d[10] & 7)) if d[10] & 0x80 else 0)]) + b"\x3b"


def test_malformed_files_are_corrupt_input(L):
    base = dict(CASES)["disposal_mix"]
    for why, data in _mutations(base):
        with pytest.raises(L.B200Error) as e:
            L.gif_decode(data)
        assert e.value.code == L.ERR_CORRUPT_INPUT, why


def test_bad_codes_are_corrupt_input(L):
    idx = np.arange(12, dtype=np.uint8).reshape(3, 4) % 4
    good = gif_cases.raw_gif(4, 3, [dict(x=0, y=0, idx=idx, table=[(0, 0, 0)] * 4, m=2)])
    L.gif_decode(good)
    i = good.index(b"\x2c") + 10 + 3 * 4
    # CLEAR then a code past the dictionary (7 at width 3), and a stream that ends before the pixels do
    for data, why in ((good[:i] + b"\x02\x01\x3c\x00\x3b", "code past dictionary"), (good[:i] + b"\x02\x01\x0c\x00\x3b", "too short"),
                      (good[:i] + b"\x02\x02\x2c\x00\x00\x3b", "index past table")):
        with pytest.raises(L.B200Error) as e:
            L.gif_decode(data)
        assert e.value.code == L.ERR_CORRUPT_INPUT, why


def test_frame_past_the_screen_is_unsupported(L):
    f = dict(x=3, y=0, idx=np.zeros((2, 4), np.uint8), table=[(0, 0, 0), (1, 1, 1)], m=2)
    with pytest.raises(L.B200Error) as e:
        L.gif_decode(gif_cases.raw_gif(6, 2, [f]))
    assert e.value.code == L.ERR_UNSUPPORTED


@pytest.mark.parametrize("seg", [GIF_SEG, 64, 5])
def test_lzw_walk_decodes_back_around_segment_boundaries(emul, seg):
    rng = np.random.default_rng(seg)
    for m in (2, 5, 8):
        for n in (1, 2, seg - 1, seg, seg + 1, 2 * seg, 3 * seg + 7):
            for kind in ("random", "runs"):
                if kind == "random":
                    idx = rng.integers(0, 1 << m, n).astype(np.uint8)
                else:
                    idx = np.repeat(rng.integers(0, 1 << m, n // 7 + 1), 7)[:n].astype(np.uint8)
                out = unblock(emul_lzw(emul, idx, m, seg))
                assert gifutil.lzw_decode(out, m, n) == idx.tobytes(), (m, n, kind)


def test_lzw_walk_fills_the_dictionary_inside_a_segment(emul):
    rng = np.random.default_rng(9)
    idx = rng.integers(0, 256, 3 * GIF_SEG + 11).astype(np.uint8)
    out = unblock(emul_lzw(emul, idx, 8, GIF_SEG))
    assert gifutil.lzw_decode(out, 8, idx.size) == idx.tobytes()


def test_lzw_twin_is_the_walk(emul):
    from oracle import gif as G
    rng = np.random.default_rng(3)
    for n in (1, GIF_SEG - 1, GIF_SEG, GIF_SEG + 1, 5 * GIF_SEG + 3):
        idx = rng.integers(0, 32, n).astype(np.uint8)
        assert G.gif_lzw(idx, 5) == emul_lzw(emul, idx, 5, GIF_SEG)


def test_quantiser_twin_without_exact_path_is_the_png_twin_above_256_values(O):
    """orc_gif_quantize restates orc_png_quantize's non-exact path: on images with more than 256 values both take it"""
    from oracle import gif as G
    from oracle.png_quant import png_quantize
    rng = np.random.default_rng(4)
    for h, w, clear in ((23, 37, False), (40, 64, True), (1, 300, False)):
        img = rng.integers(0, 256, (h, w, 4)).astype(np.uint8)
        img[..., 3] = 255
        if clear:
            img[:, : w // 5] = 0
        for q in (1, 50, 80, 100):
            a, b = G.gif_quantize(img, q), png_quantize(img, q)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (h, w, q)


def test_quantiser_twin_without_exact_path_quantises_few_values(O):
    from oracle import gif as G
    rng = np.random.default_rng(6)
    img = np.zeros((30, 40, 4), np.uint8)
    img[..., :3] = rng.integers(0, 8, (30, 40, 1)) * 30
    img[..., 3] = 255
    pal, idx = G.gif_quantize(img, 1)
    assert len(pal) < 8
    assert np.all(pal[:, 3] == 255)


def _distinct_canvases(frames):
    keep = []
    for c, d in frames:
        if keep and np.array_equal(keep[-1][0], c):
            keep[-1][1] = min(keep[-1][1] + d, 65535)
        else:
            keep.append([c, d])
    return keep


def _twin(data, q):
    from oracle import gif as G
    frames, loop = gifutil.decode(data)
    canv = np.stack([c for c, _ in frames])
    return G.gif_encode(canv, [d for _, d in frames], -1 if loop is None else loop, q), frames, loop


@pytest.mark.parametrize("name,data", CASES, ids=IDS)
def test_twin_at_quality_100_shows_the_input(O, name, data):
    out, frames, loop = _twin(data, 100)
    shown, loop_out = gifutil.decode(out)
    keep = _distinct_canvases(frames)
    assert loop_out == loop
    assert sum(d for _, d in shown) == sum(d for _, d in frames) or sum(d for _, d in frames) > 65535
    assert len(shown) == len(keep)
    for (s, d), (c, dk) in zip(shown, keep):
        assert d == dk
        if len(np.unique(c.reshape(-1, 4), axis=0)) <= 256:
            assert np.array_equal(s, c), name
    info = gifutil.parse(out)
    assert all(f["disposal"] in (1, 2) and not f["interlaced"] for f in info["frames"])


@pytest.mark.parametrize("q", [1, 50, 80])
@pytest.mark.parametrize("name,data", CASES, ids=IDS)
def test_twin_below_100_keeps_transparency_and_timing(O, name, data, q):
    out, frames, loop = _twin(data, q)
    shown, loop_out = gifutil.decode(out)
    keep = _distinct_canvases(frames)
    assert loop_out == loop and len(shown) == len(keep)
    for (s, d), (c, dk) in zip(shown, keep):
        assert d == dk
        assert np.array_equal(s[..., 3], c[..., 3])
        assert not np.any(s[s[..., 3] == 0])
        err = (s[..., :3].astype(np.int64) - c[..., :3]) ** 2
        assert err.mean() <= 3 * 2000 / 3 + 1, (name, q)


@pytest.mark.parametrize("seed", [0, 1])
def test_mutated_files_never_crash(L, seed):
    rng = np.random.default_rng(seed)
    srcs = [d for n, d in CASES if n in ("disposal_mix", "anim_disposal3", "still_m2", "still_interlaced", "noise")]
    for it in range(300):
        d = bytearray(srcs[it % len(srcs)])
        mode = it % 3
        if mode == 0:
            for _ in range(1 + int(rng.integers(0, 6))):
                d[int(rng.integers(13, len(d)))] = int(rng.integers(0, 256))
        elif mode == 1:
            d = d[:int(rng.integers(1, len(d)))]
        else:
            i = int(rng.integers(13, len(d)))
            d[i:i] = bytes(rng.integers(0, 256, int(rng.integers(1, 40))).astype(np.uint8))
        try:
            L.gif_decode(bytes(d))
        except L.B200Error as e:
            assert e.code in (L.ERR_CORRUPT_INPUT, L.ERR_UNSUPPORTED)
