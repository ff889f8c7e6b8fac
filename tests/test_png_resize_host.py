"""PNG resize leg, CPU side: the oracle twin (oracle/png_resize.py) against independent decodes and restatements, and the opt-in
header as strict C99."""
import ctypes
import ctypes.util
import io
import os
import subprocess

import numpy as np
import pytest

import png_resize_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def R(O):
    from oracle import png_resize
    return png_resize


def _pillow_planes(png, ct, trns):
    """8-bit and sub-byte sources through Pillow -> planes [ch, h, w] of the decoded type"""
    from PIL import Image
    im = Image.open(io.BytesIO(png))
    im.load()
    if ct in (0,) and not trns:
        a = np.asarray(im.convert("L"))[None]
    elif ct == 0:
        a = np.moveaxis(np.asarray(im.convert("LA")), -1, 0)
    elif ct == 4:
        a = np.moveaxis(np.asarray(im.convert("LA")), -1, 0)
    elif ct in (2, 3) and not trns:
        a = np.moveaxis(np.asarray(im.convert("RGB")), -1, 0)
    else:
        a = np.moveaxis(np.asarray(im.convert("RGBA")), -1, 0)
    return a.copy()


def _numpy_planes16(O, c):
    """16-bit sources: a big-endian read of the oracle's un-filtered rows, the key giving alpha"""
    from pngutil import idat_stream
    import zlib
    _, idat, _ = idat_stream(c["png"])
    nin = cases.NIN[c["color_type"]]
    filt = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(c["height"], -1)
    raw = O.png_unfilter(filt, nin * 2)
    v = raw.view(">u2").astype(np.uint16).reshape(c["height"], c["width"], nin)
    planes = [v[:, :, k] for k in range(nin)]
    if c["trns"]:
        key = np.frombuffer(c["trns"], ">u2")
        hit = np.all(v == key[None, None, :], axis=2)
        planes.append(np.where(hit, 0, 65535).astype(np.uint16))
    return np.stack(planes)


@pytest.mark.parametrize("ct,bd,trns", cases.LEGAL, ids=[cases.case_id(*k) for k in cases.LEGAL])
def test_expansion_matches_an_independent_decode(O, R, ct, bd, trns):
    for w, h in ((13, 9), (1, 1), (7, 1), (1, 5)):
        c = cases.make(O, ct, bd, trns, w, h, seed=ct * 100 + bd + trns)
        got = R.expand_planes(c["raw"], w, h, bd, ct, c["plte"], c["trns"])
        want = _numpy_planes16(O, c) if bd == 16 else _pillow_planes(c["png"], ct, trns)
        if ct == 0 and trns and bd < 8:       # Pillow compares the key with the scaled sample; the png crate with the unscaled one
            want[1] = np.where(c["values"][:, :, 0] == int.from_bytes(c["trns"], "big"), 0, 255)
        assert got.dtype == (np.uint16 if bd == 16 else np.uint8)
        assert np.array_equal(got, want), (w, h)
        assert R.decoded_type(ct, bd, c["trns"])[1] == got.shape[0]


def test_sub_byte_key_compares_the_unscaled_sample(O, R):
    c = cases.make(O, 0, 2, True, 11, 6, seed=4)
    got = R.expand_planes(c["raw"], 11, 6, 2, 0, b"", c["trns"])
    key = int.from_bytes(c["trns"], "big")
    v = c["values"][:, :, 0]
    assert np.array_equal(got[1], np.where(v == key, 0, 255))
    assert np.array_equal(got[0], v * 255 // 3)


def test_palette_index_past_plte_is_opaque_black(O, R):
    c = cases.make(O, 3, 4, True, 9, 4, seed=2)
    got = R.expand_planes(c["raw"], 9, 4, 4, 3, c["plte"], c["trns"])
    assert tuple(got[:, 0, 0]) == (0, 0, 0, 255)                  # index 15: past PLTE (13 entries) and past tRNS


SHAPES = [((37, 53), (13, 0)), ((64, 1024), (0, 100)), ((9, 7), (40, 0)), ((30, 20), (45, 7)), ((1, 17), (0, 40)),
          ((23, 1), (9, 1)), ((16, 12), (16, 12))]


@pytest.mark.parametrize("ct,bd,trns", [(2, 8, False), (6, 8, False), (3, 4, True), (0, 1, False), (4, 8, False)],
                         ids=lambda v: str(v))
def test_8bit_resize_is_the_trusted_plane_resize_per_channel(O, R, ct, bd, trns):
    for (w, h), (dw, dh) in SHAPES:
        c = cases.make(O, ct, bd, trns, w, h, seed=w + h)
        info, rows = R.png_resize(c["raw"], w, h, bd, ct, c["plte"], c["trns"], dw, dh)
        nw, nh = O.compute_dimensions(w, h, dw, dh)
        assert (info["width"], info["height"]) == (nw, nh)
        planes = R.expand_planes(c["raw"], w, h, bd, ct, c["plte"], c["trns"])
        ch = planes.shape[0]
        got = rows.reshape(nh, nw, ch)
        for k in range(ch):
            assert np.array_equal(got[:, :, k], O.resize_plane(planes[k], nw, nh)), ((w, h), k)


_LIBM = ctypes.CDLL(ctypes.util.find_library("m"))
_LIBM.sinf.restype, _LIBM.sinf.argtypes = ctypes.c_float, [ctypes.c_float]


def _weights(n_in, n_out):
    """image 0.25.9 sample.rs tap windows, restated in float32 numpy (sequential sums, no FMA).  The sine is the C library's sinf,
    which the device's host-side tables call too: it is not always the correctly rounded value."""
    f = np.float32
    ratio = f(n_in) / f(n_out)
    sratio = max(ratio, f(1.0))
    support = f(3.0) * sratio
    out = []
    for o in range(n_out):
        x = (f(o) + f(0.5)) * ratio
        left = int(min(max(np.floor(x - support), 0), n_in - 1))
        right = int(min(max(np.ceil(x + support), left + 1), n_in))
        x = f(x - f(0.5))
        ws = []
        for i in range(left, right):
            t = f(f(f(i) - x) / sratio)
            if abs(t) < 3.0:
                def sinc(u):
                    a = f(u * f(np.pi))
                    return f(1.0) if u == 0 else f(f(_LIBM.sinf(float(a))) / a)
                ws.append(f(sinc(t) * sinc(f(t / f(3.0)))))
            else:
                ws.append(f(0.0))
        s = f(0.0)
        for wv in ws:
            s = f(s + wv)
        out.append((left, [f(wv / s) for wv in ws]))
    return out


def _resize16(plane, nw, nh):
    """independent u16 Lanczos3: vertical pass into float32, then horizontal, clamp to [0, 65535], round half away from zero"""
    h, w = plane.shape
    if (nw, nh) == (w, h):
        return plane.copy()
    f = np.float32
    src = plane.astype(np.float32)
    tmp = np.zeros((nh, w), np.float32)
    for oy, (l, ws) in enumerate(_weights(h, nh)):
        acc = np.zeros(w, np.float32)
        for i, wv in enumerate(ws):
            acc = (acc + (src[l + i] * f(wv)).astype(np.float32)).astype(np.float32)
        tmp[oy] = acc
    out = np.zeros((nh, nw), np.uint16)
    for ox, (l, ws) in enumerate(_weights(w, nw)):
        acc = np.zeros(nh, np.float32)
        for i, wv in enumerate(ws):
            acc = (acc + (tmp[:, l + i] * f(wv)).astype(np.float32)).astype(np.float32)
        acc = np.clip(acc, 0, 65535).astype(np.float64)
        out[:, ox] = (np.sign(acc) * np.floor(np.abs(acc) + 0.5)).astype(np.uint16)
    return out


@pytest.mark.parametrize("ct,trns", [(0, False), (0, True), (2, False), (2, True), (4, False), (6, False)], ids=lambda v: str(v))
def test_16bit_resize_equals_an_independent_restatement(O, R, ct, trns):
    for (w, h), (dw, dh) in SHAPES:
        c = cases.make(O, ct, 16, trns, w, h, seed=3 * w + h)
        info, rows = R.png_resize(c["raw"], w, h, 16, ct, c["plte"], c["trns"], dw, dh)
        nw, nh = info["width"], info["height"]
        assert info["bit_depth"] == 16 and info["row_bytes"] == nw * info["channels"] * 2
        planes = R.expand_planes(c["raw"], w, h, 16, ct, c["plte"], c["trns"])
        got = rows.view(">u2").reshape(nh, nw, info["channels"])
        for k in range(info["channels"]):
            assert np.array_equal(got[:, :, k], _resize16(planes[k], nw, nh)), ((w, h), k)


def test_16bit_resize_clamps_at_both_ends(R):
    step = np.zeros((12, 12), np.uint16)
    step[:, 6:] = 65535                                           # Lanczos lobes overshoot on both sides of the edge
    got = R.resize_plane_u16(step, 29, 12)
    assert got.min() == 0 and got.max() == 65535
    assert np.array_equal(got, _resize16(step, 29, 12))


def test_opt_in_header_is_c99(L, tmp_path):
    src = tmp_path / "png_resize_abi.c"
    src.write_text('#include "b200_caesium_png_resize.h"\n'
                   "typedef void (*fn)(void);\n"
                   "int main(void) { fn f[2] = {(fn)b200_set_png_resize, (fn)b200_png_resize_samples}; return f[0] == 0 || f[1] == 0 || b200_set_png_resize(2) == 0; }\n")
    pkg = os.path.join(ROOT, "caesium-clt_b200")
    exe = str(tmp_path / "png_resize_abi")
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", exe,
                        "-L", pkg, "-lb200caesium", "-Wl,-rpath," + pkg], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert subprocess.run([exe]).returncode == 0
